/*
 * kai_engine.h — C ABI of libkaigpu.so, the H100-native scheduling-cycle engine.
 *
 * This is the drop-in boundary for ONE hot path of NVIDIA/KAI-Scheduler: the
 * per-Session scheduling cycle in pkg/scheduler.  A Go `framework.Action`
 * (reference: pkg/scheduler/framework/interface.go:41-47, registered through
 * framework.RegisterAction, pkg/scheduler/framework/plugins.go:47-62) packs
 * `ssn.ClusterInfo` into the structure-of-arrays snapshot below, calls
 * kai_engine_run(), and replays the returned bindings through
 * Statement.Allocate/Pipeline/Evict + Commit (INTEGRATION.md shows the cgo stub).
 *
 * Conventions
 *   - plain C, no exceptions cross the boundary; every call returns 0 (KAI_OK)
 *     or a negative kai_status; kai_last_error() gives a message.
 *   - the caller owns every input buffer; buffers only have to stay valid for
 *     the duration of kai_engine_load_snapshot() (the engine copies to pinned
 *     host memory and then to HBM).
 *   - result arrays are engine-owned and valid until the next
 *     kai_engine_load_snapshot()/kai_engine_run()/kai_engine_destroy().
 *   - one caller thread at a time per engine (Scheduler.runOnce is
 *     single-threaded: pkg/scheduler/scheduler.go:107-138).
 *   - there is NO CPU fallback inside the library: if no CUDA device is
 *     usable, kai_engine_create() fails with KAI_ERR_NO_DEVICE and the shim
 *     falls back to the stock Go action for that cycle.
 *
 * Resource vector layout (reference: api/resource_info/resource_vector.go:23-36):
 *   index 0 cpu (milli-cores), 1 memory (bytes), 2 gpu (whole devices),
 *   3 pods, 4.. extra scalar resources in first-seen order.
 * Queue-level resource order (reference: plugins/proportion/resource_share/
 *   resource_quantities.go `AllResources`): 0 CPU, 1 Memory, 2 GPU.
 */
#ifndef KAI_ENGINE_H_
#define KAI_ENGINE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KAI_ABI_VERSION 7
#define KAI_MAX_RES 8 /* resource dims per node/task row (>= 4) */
#define KAI_QRES 3    /* queue-level resources: CPU, Memory, GPU */
#define KAI_MAX_QUEUE_DEPTH 8 /* max levels in the queue hierarchy */

enum { KAI_RES_CPU = 0, KAI_RES_MEM = 1, KAI_RES_GPU = 2, KAI_RES_PODS = 3 };
enum { KAI_Q_CPU = 0, KAI_Q_MEM = 1, KAI_Q_GPU = 2 };

/* reference: pkg/common/constants/constants.go:8-13 */
#define KAI_UNLIMITED (-1.0)

typedef enum kai_status {
  KAI_OK = 0,
  KAI_ERR_INVALID = -1,     /* bad argument / malformed snapshot */
  KAI_ERR_NO_DEVICE = -2,   /* no usable CUDA device (no CPU fallback exists) */
  KAI_ERR_CUDA = -3,        /* CUDA runtime error, see kai_last_error */
  KAI_ERR_UNSUPPORTED = -4, /* snapshot uses a feature outside the engine's scope */
  KAI_ERR_STATE = -5        /* call order violated (e.g. run before load) */
} kai_status;

/* Pod status bitmask values. reference: api/pod_status/pod_status.go:25-71 */
enum {
  KAI_POD_PENDING = 1,
  KAI_POD_GATED = 2,
  KAI_POD_ALLOCATED = 4,
  KAI_POD_PIPELINED = 8,
  KAI_POD_BINDING = 16,
  KAI_POD_BOUND = 32,
  KAI_POD_RUNNING = 64,
  KAI_POD_RELEASING = 128,
  KAI_POD_SUCCEEDED = 256,
  KAI_POD_FAILED = 512,
  KAI_POD_UNKNOWN = 1024,
  KAI_POD_DELETED = 2048
};

/* node_flags bits */
enum {
  KAI_NODE_READY = 1u,       /* counts toward fair-share totals (proportion.go:258-263) */
  KAI_NODE_NOT_CPU_ONLY = 2u /* MIG-enabled or DRA GPUs: never a "CPU-only node" (node_info.go:697-702) */
};

/* job_flags bits */
enum {
  KAI_JOB_PREEMPTIBLE = 1u /* pkg/common/podgroup/preemptible.go:10-26 */
};

/* Actions. reference: pkg/scheduler/framework/interface.go:30-39 */
typedef enum kai_action {
  KAI_ACTION_ALLOCATE = 1,
  KAI_ACTION_CONSOLIDATION = 2,
  KAI_ACTION_RECLAIM = 3,
  KAI_ACTION_PREEMPT = 4,           /* actions/preempt/preempt.go:46-161 */
  KAI_ACTION_STALEGANGEVICTION = 5  /* actions/stalegangeviction/stalegangeviction.go:29-95 */
} kai_action;

/* minruntime `reclaimResolveMethod` (plugins/minruntime/minruntime.go:27-29; resolver.go:83-187) */
enum { KAI_RESOLVE_LCA = 0, KAI_RESOLVE_QUEUE = 1 };

/* node placement strategy. reference: plugins/nodeplacement/nodeplacement.go:53-73 */
enum { KAI_PLACEMENT_BINPACK = 0, KAI_PLACEMENT_SPREAD = 1 };

typedef struct kai_config {
  int32_t abi_version;          /* = KAI_ABI_VERSION */
  int32_t device;               /* CUDA device ordinal */
  int32_t gpu_placement;        /* nodeplacement `gpu:` argument */
  int32_t cpu_placement;        /* nodeplacement `cpu:` argument */
  double k_value;               /* proportion `kValue` (proportion.go:78-85) */
  double saturation_multiplier; /* proportion `relcaimerSaturationMultiplier` (proportion.go:68-76) */
  int32_t max_consolidation_preemptees; /* -1 = unlimited (options.go:38) */
  int32_t allow_consolidating_reclaim;  /* options.go:121 */
  /* node sharding across engines of one box (SURVEY §8e).  shard_count = 1 for a single GPU.  Shard s owns the nodes
     of name rank s, s + S, s + 2S, ... (kai_shard_range); the exchange segment is wired with kai_engine_wire_peers(). */
  int32_t shard_rank;
  int32_t shard_count;
  /* SchedulerParams.UseSchedulingSignatures (cmd/scheduler/app/options/options.go:120; production default true, the
     reference's action tests run with false): reclaim / consolidation skip jobs that are "not easier to schedule" than
     a job with the same kai_snapshot.job_signature that already failed (actions/common/minimal_job_comparison.go). */
  int32_t use_scheduling_signatures;
  /* SchedulerParams.GlobalDefaultStalenessGracePeriod in seconds: < 0 = stale gangs are never evicted, 0 = evicted in
     the cycle that finds them stale; > 0 = evicted once `now_s - job_stale_since_s >= grace` (a job without a staleness
     timestamp has just turned stale: not yet).  Production default 60 (cmd/scheduler/app/options/options.go). */
  int32_t staleness_grace_period_s;
  /* minruntime plugin arguments (plugins/minruntime/minruntime.go:24-78): `defaultReclaimMinRuntime`,
     `defaultPreemptMinRuntime` in seconds (negative or unparsable = 0) and `reclaimResolveMethod`. */
  int32_t reclaim_resolve_method; /* KAI_RESOLVE_LCA (default) or KAI_RESOLVE_QUEUE */
  double default_reclaim_min_runtime_s;
  double default_preempt_min_runtime_s;
} kai_config;

/*
 * Structure-of-arrays snapshot of api.ClusterInfo
 * (reference: pkg/scheduler/api/cluster_info.go:43-64).
 *
 * Node tables are resource-major: x[r * n_nodes + n].
 * Queue tables are resource-major as well: x[r * n_queues + q], r in KAI_Q_*.
 * Task request table is task-major: task_req[t * n_res + r].
 */
typedef struct kai_snapshot {
  int32_t abi_version;
  int32_t n_res; /* 4..KAI_MAX_RES */
  int32_t n_nodes;
  int32_t n_queues;
  int32_t n_jobs;
  int32_t n_podsets;
  int32_t n_tasks;
  int32_t n_pred_classes;

  /* ---- nodes: NodeInfo (api/node_info/node_info.go:68-105) ---- */
  const double *node_allocatable; /* [n_res][N] Allocatable */
  const double *node_idle;        /* [n_res][N] Idle */
  const double *node_releasing;   /* [n_res][N] Releasing */
  const int32_t *node_name_rank;  /* [N] rank of Name in byte-wise ascending order (session.go:480-485) */
  const uint32_t *node_flags;     /* [N] KAI_NODE_* */
  const double *node_gpu_count;   /* [N] GetNumberOfGPUsInNode (node_info.go:644-651); NULL = Allocatable gpu */
  const double *node_foreign;     /* [3][N] resources of active pods of other schedulers (proportion.go:276-286); NULL = 0 */

  /* ---- queues: QueueInfo (api/queue_info/queue_info.go:32-43) ---- */
  const int32_t *queue_parent;   /* [Q] index of ParentQueue, -1 = top level */
  const int32_t *queue_priority; /* [Q] */
  const int64_t *queue_creation; /* [Q] CreationTimestamp, any monotone integer clock */
  const int32_t *queue_uid_rank; /* [Q] rank of UID string */
  const double *queue_deserved;  /* [3][Q] quota; memory already in bytes; -1 unlimited */
  const double *queue_limit;     /* [3][Q] limit; -1 unlimited */
  const double *queue_oqw;       /* [3][Q] overQuotaWeight */
  const double *queue_usage;     /* [3][Q] historical usage (normalised); NULL = 0 */

  /* ---- jobs: PodGroupInfo (api/podgroup_info/job_info.go:65-103) ---- */
  const int32_t *job_queue;        /* [J] leaf queue index, -1 = queue missing */
  const int32_t *job_priority;     /* [J] */
  const int32_t *job_order_rank;   /* [J] rank under (CreationTimestamp, UID) (session_plugins.go:235-241) */
  const uint32_t *job_flags;       /* [J] KAI_JOB_* */
  const int32_t *job_podset_begin; /* [J+1] podsets of job j = [begin[j], begin[j+1]), in PodSet name order */

  /* ---- podsets: subgroup_info.PodSet ---- */
  const int32_t *podset_min_available; /* [S] */
  const int32_t *podset_task_begin;    /* [S+1] tasks of podset s = [begin[s], begin[s+1]) */

  /* ---- tasks: PodInfo (api/pod_info/pod_info.go:70-112) ---- */
  const int32_t *task_status;     /* [T] KAI_POD_* */
  const int32_t *task_node;       /* [T] node index for active-used tasks, else -1 */
  const double *task_req;         /* [T][n_res] ResReq vector; pods column = 1 (pod_info.go:390) */
  const int32_t *task_order_rank; /* [T] rank under TaskOrderFn within the job (session_plugins.go:244-259) */
  const int32_t *task_nominated;  /* [T] Status.NominatedNodeName as node index, -1 none; NULL = none */
  const int32_t *task_pred_class; /* [T] row of pred_mask, -1 = passes everywhere; NULL = all -1 */

  /* ---- host-evaluated predicates (k8s Filters, node conditions, MIG rules):
         bit n of row c set = node n passes for predicate class c ---- */
  const uint32_t *pred_mask; /* [n_pred_classes][(N+31)/32] */

  /* ---- PodGroupInfo.GetSchedulingConstraintsSignature (job_info.go:547-570) as a class id: jobs with equal
         signatures get equal ids; -1 = unique.  NULL = all -1. ---- */
  const int32_t *job_signature; /* [J] */

  /* ---- Topology CRs (pkg/apis/kai/v1alpha1 Topology; plugins/topology/topology_plugin.go:57-110).
         Levels of topology k = [topology_level_begin[k], topology_level_begin[k+1]) in Spec.Levels order (top level
         first).  node_domain[l][n] = the node's domain at level l: dense ids per level assigned in ascending
         DomainID order (DomainID = the label values of the levels down to l joined by ".", topology_structs.go:76-82),
         -1 = the node lacks that label (a node missing any level is outside the topology, common.go:63-70).
         Constraints of the job's root SubGroupSet (api/topology_info): job_topology[j] = topology index or -1,
         job_required_level / job_preferred_level = level index inside that topology (0 = top) or -1. ---- */
  int32_t n_topologies;
  int32_t reserved1;
  const int32_t *topology_level_begin; /* [n_topologies + 1] */
  const int32_t *node_domain;          /* [n_levels_total][N] */
  const int32_t *job_topology;         /* [J]; NULL = no constraints */
  const int32_t *job_required_level;   /* [J] */
  const int32_t *job_preferred_level;  /* [J] */

  /* ---- SubGroupSet tree of every job (api/podgroup_info/subgroup_info/subgroupset.go; allocate.go:36-83 walks it).
         Sets of job j = [job_sgs_begin[j], job_sgs_begin[j+1]); the first one is the root.  NULL job_sgs_begin =
         every job has only its root set holding all its PodSets, with the job_* constraint above and no PodSet
         constraints.  When given, the root's constraint is sgs_* of its entry and job_* are ignored. ---- */
  int32_t n_subgroup_sets;
  int32_t reserved2;
  const int32_t *job_sgs_begin;          /* [J+1] */
  const int32_t *sgs_parent;             /* [G] global index of the parent set, -1 for a root */
  const int32_t *sgs_name_rank;          /* [G] rank of the set's name among the sets of its job (SubGroupSetOrderFn) */
  const int32_t *sgs_topology;           /* [G] topology index, -1 none */
  const int32_t *sgs_required_level;     /* [G] */
  const int32_t *sgs_preferred_level;    /* [G] */
  const int32_t *podset_sgs;             /* [S] global index of the set that holds the PodSet */
  const int32_t *podset_topology;        /* [S] PodSet's own constraint, -1 none; NULL = none */
  const int32_t *podset_required_level;  /* [S] */
  const int32_t *podset_preferred_level; /* [S] */

  /* ---- min-runtime protection of victims (plugins/minruntime): a non-elastic job whose LastStartTimestamp + the
         resolved min-runtime lies after `now_s` is not offered as a reclaim / preempt victim; an elastic one may only
         shrink to its minAvailable.  Durations in seconds, < 0 = not set on that queue (QueueSpec.PreemptMinRuntime /
         ReclaimMinRuntime are pointers, pkg/apis/scheduling/v2/queue_types.go:40-46); job_last_start_s <= 0 = never
         started (PodGroupInfo.LastStartTimestamp nil or zero).  NULL arrays = nothing set. ---- */
  double now_s;                              /* the reference reads time.Now() at every check; one instant per cycle here */
  const double *queue_preempt_min_runtime_s; /* [Q] */
  const double *queue_reclaim_min_runtime_s; /* [Q] */
  const double *job_last_start_s;            /* [J] seconds on the clock of now_s */
  /* ---- stale gangs (actions/stalegangeviction/stalegangeviction.go:42-62): PodGroupInfo.StalenessInfo.TimeStamp, read
         from the PodGroup's `kai.scheduler/stale-podgroup-timestamp` annotation (job_info.go:174-182), on the clock of
         now_s; <= 0 = nil (the action stamps time.Now(), i.e. zero time in stale state).  NULL = nil for all jobs. ---- */
  const double *job_stale_since_s;           /* [J] */
  /* ---- resident snapshot (ABI v7).  The reference rebuilds ClusterInfo from the informer caches every cycle
         (cache/cluster_info/cluster_info.go:118-228) although most of it — queues, pod groups, PodSets, requests, order
         ranks, node identities and labels — only changes when an object is added, removed or edited.  A caller that
         tracks that (the informers' resourceVersions) passes the same non-zero structure_epoch as long as only the
         per-cycle columns changed:
           node_idle, node_releasing, node_flags, node_foreign, queue_usage, task_status, task_node, task_nominated,
           now_s, job_last_start_s, job_stale_since_s.
         kai_engine_load_snapshot then keeps everything it derived from the rest (index structures, task renumbering,
         device copies) and uploads those columns only.  0 = always a full load.  Every other field is structural and
         must still describe the same cluster (it is not re-read): the caller bumps the epoch when an object is added or
         removed, when a spec changes, and also on these status changes of a node: its allocatable resources or GPU
         count (node_allocatable, node_gpu_count) and the conditions or taints that feed pred_mask / task_pred_class.
         A change in the count or presence of any array (the shape) falls back to a full load by itself.
         KAI_RESIDENT_CHECK=1 makes a resident load compare checksums of every structural array with the last full
         load and fail with KAI_ERR_INVALID naming the first field that changed (off by default; a test aid). ---- */
  uint64_t structure_epoch;
} kai_snapshot;

/* One entry per job popped by an action, in visiting order. */
typedef struct kai_job_visit {
  int32_t job;
  int32_t outcome; /* 1 = statement committed, 0 = discarded */
} kai_job_visit;

typedef struct kai_result {
  int32_t n_tasks;
  const int32_t *task_node;   /* [T] node index after the action, -1 = none */
  const int32_t *task_status; /* [T] KAI_POD_* after the action (Binding for committed allocations) */
  int32_t n_visits;
  const kai_job_visit *visits; /* [n_visits] */
  int32_t n_queues;
  const double *queue_fair_share;              /* [3][Q] */
  const double *queue_allocated;               /* [3][Q] */
  const double *queue_allocated_non_preemptible; /* [3][Q] */
  const double *queue_request;                 /* [3][Q] */
  const double *total_resource;                /* [3] */
  int32_t n_nodes;
  const double *node_idle;      /* [n_res][N] after the action */
  const double *node_releasing; /* [n_res][N] after the action */
  int64_t pods_placed;          /* tasks that moved Pending -> Binding/Pipelined in this run */
  int64_t pods_evicted;         /* tasks that moved to Releasing in this run */
} kai_result;

typedef struct kai_stats {
  double upload_ms;      /* host -> HBM snapshot copy of the last load */
  double open_session_ms;/* totals + queue usage + fair-share kernels */
  double action_ms;      /* device time of the last kai_engine_run action kernel (CUDA events) */
  double download_ms;    /* HBM -> host result copy */
  int64_t decisions;     /* node-table sweeps executed (one per allocateTask call) */
  int64_t nodes_scanned; /* sum over sweeps of node-set size */
  int64_t kernel_launches; /* kernels launched by the last load+run */
  int64_t algorithmic_bytes; /* nodes_scanned * bytes/node (DESIGN.md) */
} kai_stats;

typedef struct kai_engine kai_engine;

/* replaces: the per-cycle construction in framework.OpenSession
   (pkg/scheduler/framework/framework.go:32-62) for the plugins on the path. */
int kai_engine_create(const kai_config *cfg, kai_engine **out);

/* replaces: cache.Snapshot() -> ClusterInfo hand-off (framework/session.go:341-366)
   followed by proportion.OnSessionOpen (plugins/proportion/proportion.go:99-124):
   copies the SoA to HBM and computes totals, queue usage and fair shares. */
int kai_engine_load_snapshot(kai_engine *e, const kai_snapshot *snap);

/* replaces: Action.Execute(ssn) of the default action list
   (actions/allocate/allocate.go:46-111, actions/consolidation/consolidation.go:32-106,
   actions/reclaim/reclaim.go:46-119, actions/preempt/preempt.go:46-123,
   actions/stalegangeviction/stalegangeviction.go:29-95).  Session state persists between calls so that
   `allocate, consolidation, reclaim, preempt, stalegangeviction` run in sequence on one loaded snapshot.
   Errors: KAI_ERR_UNSUPPORTED for inputs the engine does not run (KAI_TRANSPORT=persistent or KAI_SEQUENCER=device
   in the environment: modes it no longer has); the session is then unchanged and the caller runs the stock action. */
int kai_engine_run(kai_engine *e, kai_action action, kai_result *out);

/* replaces: fairshare-simulator's SetResourcesShare call
   (cmd/fairshare-simulator/main.go:95-103) — results of the last load. */
int kai_engine_fair_share(kai_engine *e, kai_result *out);

int kai_engine_stats(kai_engine *e, kai_stats *out);

/* Measurement aid (no reference counterpart): times `n_launches` back-to-back launches of the sweep kernel (k_record,
   one list sweep of a 1-GPU / 1000 mCPU / 1e9 B pod over every node row of the loaded snapshot: the a4-a8 inner loop
   of framework/session.go:201-264) and then as many of the merge kernel (k_merge: sort, cut and stream one answer
   list to host memory) with CUDA events on the engine's stream.  The session state is not changed.  Writes the elapsed
   milliseconds of both and the node rows one launch sweeps (x 76 B = its algorithmic bytes, SURVEY.md 8d). */
int kai_engine_time_sweeps(kai_engine *e, int n_launches, double *elapsed_ms, double *merge_ms, int64_t *rows_per_launch);

/* Multi-GPU wiring (one engine per process per GPU, SURVEY.md §8e).  Shard s of
   shard_count owns the nodes of name rank s, s + S, s + 2S, ... (kai_shard_range
   returns first_rank = s and their count): consecutive ranks sit on different GPUs
   and different scanners, so the best rows of a sweep come from many scanners.  The reduced answer line of
   every GPU lives in one shared host segment: rank 0 creates it and exports its
   64-byte handle; after an out-of-band broadcast/all-gather (torch.distributed,
   MPI, ...) every rank passes the handle table (entry 0 is read) to
   kai_engine_wire_peers.  Results: task bindings / queue tables are identical on
   all ranks; node tables are valid for the rank's own rows. */
#define KAI_PEER_HANDLE_BYTES 64
int kai_engine_export_peer_handle(kai_engine *e, uint8_t handle[KAI_PEER_HANDLE_BYTES]);
int kai_engine_wire_peers(kai_engine *e, const uint8_t *handles /* [shard_count][64] */);
int kai_shard_range(int n_nodes, int shard_count, int shard_rank, int *first_rank, int *count);

void kai_engine_destroy(kai_engine *e);
const char *kai_last_error(const kai_engine *e);
int kai_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* KAI_ENGINE_H_ */
