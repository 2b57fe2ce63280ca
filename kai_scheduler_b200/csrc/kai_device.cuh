// kai_device.cuh — device-side data layout shared by the kernels of libkaigpu.so.
//
// HBM layout (DESIGN.md §3):
//   node tables   resource-major f64 [R][N]  (allocatable, idle, releasing) + name_rank/flags [N]
//   queue tables  resource-major f64 [3][Q]
//   task request  task-major f64 [T][R]
//   session state (one copy): task status/node/virtual, queue allocated, node idle/releasing
//   replica state (one copy per CTA of the persistent action kernel): the mutable part of the
//     session that the replicated sequencer (thread 0 of every CTA) updates in lock step
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/kai_engine.h"

namespace kai {

constexpr int QR = KAI_QRES;
constexpr int kThreads = 128;          // threads per CTA of the action kernel (4 warps: cheap barriers/reductions)
constexpr int kMaxGrid = 1024;         // exchange slots per GPU
constexpr uint32_t kNoRank = 0xFFFFFFFFu;
constexpr int kDecWords = 16;         // tagged words of one decision record
constexpr int kMaxDelta = 256;        // node deltas carried by one decision record
constexpr int kTopM = 4;              // candidates every scanner returns per sweep (host-sequenced mode)
constexpr int kListScanners = 2048;   // scanners of all GPUs of a box (list lines in host memory)
constexpr int kListLineWords = 8;     // one 64-byte line = 4 tagged words
constexpr int kListLines = 1 + kTopM; // line 0: the M candidate words, lines 1..M: row values of candidate m
constexpr int kMaxDomLevels = 8;      // topology levels of all Topology CRs together (rows keep one domain id per level)
constexpr int kDomBuckets = 4096;     // preferred-level domains that can carry a node score at a time

constexpr int kActiveUsed = KAI_POD_ALLOCATED | KAI_POD_PIPELINED | KAI_POD_BINDING | KAI_POD_BOUND |
                            KAI_POD_RUNNING | KAI_POD_RELEASING;
constexpr int kActiveAllocated =
    KAI_POD_ALLOCATED | KAI_POD_PIPELINED | KAI_POD_BINDING | KAI_POD_BOUND | KAI_POD_RUNNING;
constexpr int kAlive = kActiveAllocated | KAI_POD_PENDING | KAI_POD_GATED;
constexpr int kAllocatedStatuses = KAI_POD_ALLOCATED | KAI_POD_BOUND | KAI_POD_BINDING | KAI_POD_RUNNING;

struct Op {  // framework/statement.go operations (allocate / pipeline / evict / undo)
  int kind, task, prev_status, prev_node, next_node, prev_virtual, undo_index, pad;
};
enum { OP_ALLOCATE = 0, OP_PIPELINE = 1, OP_EVICT = 2, OP_UNDO = 3 };

// queue-node flags of the job-order tree (actions/utils/job_order_by_queue.go:18-25)
enum { QN_EXISTS = 1, QN_LINKED = 2, QN_REORDER = 4 };

// Per-job record written by k_prep_jobs (one 64-byte line): everything the sequencer needs to pop, admit
// and allocate a job whose tasks have not been touched yet in this action.
struct __align__(64) JobRec {
  double req0[3];  // GetTasksToAllocateInitResource at action start (valid when n_podsets == 1)
  int n_tta;       // >= 0: GetTasksToAllocate is exactly tasks [tb, tb + n_tta) (all pending); -1: general path
  int tb;          // first task of podset ps0
  int ps0;         // first podset
  int n_podsets;
  int cnt[3];      // podset ps0: active-allocated, pending, pipelined task counts at action start
  int pad[3];
};

// Order-independence test of the open-session sums (k_node_totals / k_queue_usage), zeroed by every load.
// Index 0 = node totals, 1 = queue usage.
struct OpenSums {
  unsigned long long sum_abs[2][3];  // per resource: sum of |summand| over the integer-valued summands (saturating)
  unsigned int inexact[2];           // bit r: resource r has a summand that is not an integer of at most 2^53
  unsigned int blocks_done[2];       // last-block ticket
};

// Immutable (per cycle) device snapshot + session state pointers.  Passed by value to kernels.
struct DevSnap {
  int R, N, Q, J, S, T, NPC, mask_words;
  int n_top, max_job_tasks, max_job_podsets, n_levels;
  // nodes
  const double *alloc;      // [R][N]
  double *idle, *rel;       // [R][N] session state
  const int *name_rank;     // [N]
  const int *rank_to_node;  // [N]
  const uint32_t *nflags;   // [N]
  const double *gpu_count;  // [N]
  const double *foreign;    // [3][N] or null
  // queues
  const int *q_parent, *q_priority, *q_uid_rank, *q_nchildren;
  const long long *q_creation;
  const double *q_deserved, *q_limit, *q_oqw, *q_usage;  // [3][Q]
  double *q_fair, *q_request;                            // [3][Q] computed by open-session kernels
  double *q_alloc, *q_alloc_np;                          // [3][Q] session state
  const int *q_child_begin, *q_children;                 // CSR of children (ascending index)
  const int *top_queues;                                 // [n_top]
  const int *level_group_begin, *level_groups;           // fair-share: groups (parent queue or -1) per level
  const int *q_task_begin, *q_tasks;                     // CSR: device indices of the tasks under each queue, caller order
  const int *q_job_begin;                                // [Q+1] leaf-heap arena offsets
  const int *q_jobs_sorted;                              // [J] jobs grouped by queue, (priority desc, order_rank)
  // jobs
  const int *j_queue, *j_priority, *j_order_rank, *j_ps_begin;
  const uint32_t *j_flags;
  // podsets
  const int *ps_min, *ps_task_begin, *ps_job;
  // tasks
  const double *t_req;  // [T][R]
  const int *t_job, *t_podset, *t_nominated, *t_pred_class;
  int *t_status, *t_node, *t_node_status;  // session state
  unsigned char *t_virtual;                // session state
  const uint32_t *pred_mask;
  double *total;  // [3] device
  OpenSums *osum;
  // ---- written by the fair-share / prepare kernels (device only) ----
  double *q_allocatable;  // [3][Q] GetAllocatableShare per queue (static within a cycle)
  unsigned long long *j_key0;  // [J] JobOrderFn sort key at action start
  int *leaf_sorted;            // [J] eligible jobs per leaf queue (arena offsets q_job_begin) in JobOrderFn order
  int *leaf_count;             // [Q]
  int *ps_cnt0;                // [3][S] tasks per podset: active-allocated, pending, pipelined
  double *j_req;               // [J][3] cached GetTasksToAllocateInitResource
  unsigned char *j_req_valid;  // [J]
  Op *ops;                     // [ops_cap] statement log
  int *tta;                    // [max_job_tasks + 1]
  int *ps_order;               // [max_job_podsets + 1]
  unsigned char *hot_global;   // hot arrays when they do not fit in shared memory
  JobRec *jrec;                // [J]
};

// Cached comparator inputs of one queue node (plugins/proportion/queue_order/queue_order.go:19-73)
struct QKey {
  double drf_job, drf;
  // the first four criteria of queue_order.go:19-73 packed so that an ascending integer compare orders them as the
  // comparator does: over fair share (bit 44) | not starved (43) | inverted priority (42..10) | limit violation (9)
  unsigned long long w0;
  int priority;
  unsigned char over, starved, viol, valid;
};

// Mutable state the sequencer CTA works on.  The "hot" per-queue arrays live in its shared memory when
// they fit (ActionParams.hot_in_smem), otherwise in global memory; the cold arrays are the session
// arrays in HBM/L2 themselves (single copy).
struct Replica {
  // hot: per queue
  double *q_alloc, *q_alloc_np;  // [3][Q]
  QKey *qkey;                    // [Q]
  int *leaf_head, *leaf_end;     // [Q] sorted part of the leaf job list = leaf_heap[head, end)
  int *ovl_len;                  // [Q] overflow heap (re-pushed jobs) = leaf_heap[q_job_begin, +ovl_len)
  int *child_len;                // [Q]
  int *child_heap;               // [Q] arena by q_child_begin
  int *root_heap;                // [n_top + 1]
  unsigned char *qn_flags;       // [Q]
  unsigned int *touched;         // [ceil(J/32)] jobs whose task statuses changed in this action
  // cold
  int *t_status, *t_node, *t_node_status;
  unsigned char *t_virtual;
  int *ps_active_alloc, *ps_pending, *ps_pipelined;  // [S]
  double *j_req;                                     // [J][3] cached GetTasksToAllocateInitResource
  unsigned char *j_req_valid;
  unsigned long long *j_key;  // [J]
  int *leaf_heap;             // [J]
  Op *ops;                    // [ops_cap]
  int *tta;                   // [max_job_tasks]
  int *ps_order;              // [max_job_podsets]
};

struct ActionParams {
  DevSnap s;
  kai_config cfg;
  int action;
  int grid;             // CTAs of this GPU
  int nodes_per_cta;    // node rows per CTA (tile height)
  int ops_cap;
  unsigned long long *dbuf;  // decision record: [2][kDecWords] tagged 128-bit words (sequencer -> scanners)
  unsigned long long *delta; // node delta list: [2][kMaxDelta] tagged words {name_rank(node) | code<<28 | task<<32, seq}
  unsigned long long *xbuf;  // exchange slots: [2][kMaxGrid][8] u64 (tagged 128-bit words A, B, C, D)
  unsigned long long *mmbuf; // min/max exchange: [2][kMaxGrid][8] u64
  kai_job_visit *visits;     // [visits_cap]
  int visits_cap;
  long long *counters;  // [16]: n_visits, sweeps, nodes_scanned, pods_placed, pods_evicted, minmax_exchanges, error, seq, phase timers
  unsigned int seq0;    // first exchange sequence number of this launch
  int hot_in_smem;      // hot replica arrays carved from dynamic shared memory after the node tile
  size_t tile_bytes, hot_bytes;
  int batching;         // same-node batching of consecutive identical pods (1 = on)
  int mode;             // 0 = device-resident sequencer (CTA 0), 1 = host-sequenced (CTA 0 relays host records)
  unsigned long long *h_rec, *h_delta;  // mode 1: decision record / delta words in pinned mapped host memory
  unsigned long long *h_slot, *h_mmslot;  // mode 1: this GPU's reduced answer line [2][kSlotWords] in (shared) host memory
  int spin_log2;        // watchdog: polls before a wait is declared dead
  int topm;             // mode 1: scanners answer with their kTopM best rows (0 = single best through the relay)
  unsigned long long *h_list;  // mode 1: [2][kListScanners][kListLines][kListLineWords] in (shared) host memory
  int scanner_base;     // global index of this GPU's scanner 0 in h_list
  const int *node_domain;  // [n_dom_levels][N] topology domain of every node per level (-1 = label missing), or null
  int n_dom_levels;
  // ---- launch transport (mode 2): one kernel launch per decision record, node tiles resident in global memory ----
  unsigned char *g_tiles;      // [scanners][g_tile_stride] tiles in the layout of the shared-memory tile
  size_t g_tile_stride;
  unsigned char *g_scan_state; // [scanners][kScanStateBytes]: preferred level + per-domain score buckets of each scanner
  unsigned int *ticket;        // CTAs that finished the current launch (the last one reduces the answers)
  double *mm_result;           // [4] gpu mn, gpu mx, cpu mn, cpu mx of the last MINMAX launch (read by XB_FUSED_MM sweeps)
  unsigned long long *h_clist; // this GPU's merged candidate list [2][kCListWords] in (shared) host memory
  int fused_in_kernel;         // XB_FUSED_MM sweeps exchange their extremes inside the launch (cooperative launch: all CTAs resident)
};

constexpr int kMergeCap = 1024;                      // candidates k_merge sorts, one per thread (scanners x kTopM)
constexpr int kCEntryWords = 6;                      // score, meta, Ig, Lg, Ic, Lc
constexpr int kCListWords = 2 + kMergeCap * kCEntryWords;  // header {count | more << 31, tag} + entries
constexpr int kScanStateBytes = 16 + kDomBuckets;
constexpr int kMaxDeltaL = kMaxDelta;
enum { DK_LOAD = 6 };  // launch transport: load the tiles from the session tables (first launch of an action)

// One decision record of the launch transport, passed by value in the kernel parameter space.
struct LaunchRec {
  unsigned long long dw[kDecWords];
  unsigned int seq;
  int n_delta;
  unsigned int dkey[kMaxDeltaL];    // name rank | code << 28, or an extended entry (bit 31)
  unsigned int dtask[kMaxDeltaL];
  unsigned char dcount[kMaxDeltaL]; // repeat count - 1
};

}  // namespace kai
