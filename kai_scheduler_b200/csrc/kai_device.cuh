// kai_device.cuh — device-side data layout shared by the kernels of libkaigpu.so.
//
// HBM layout (DESIGN.md §3):
//   node tables   resource-major f64 [R][N]  (allocatable, idle, releasing) + name_rank/flags [N]
//   queue tables  resource-major f64 [3][Q]
//   task request  task-major f64 [T][R]
//   session state (one copy): task status/node/virtual, queue allocated, node idle/releasing
//
// It also holds the few helpers that the kernels and the host sequencer both run (__host__ __device__): the f64
// wrappers, the job key, the tile row striping, the tracker events and the node-delta arithmetic.
#pragma once
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "../../include/kai_engine.h"

namespace kai {

constexpr int QR = KAI_QRES;
constexpr int kThreads = 128;          // threads per scanner CTA of k_record (4 warps: cheap barriers/reductions)
constexpr int kMaxGrid = 1024;         // exchange slots per GPU
constexpr uint32_t kNoRank = 0xFFFFFFFFu;
constexpr int kDecWords = 16;         // tagged words of one decision record
constexpr int kMaxDelta = 256;        // node deltas carried by one decision record
constexpr int kTopM = 4;              // candidates every scanner returns per list sweep
constexpr int kListScanners = 2048;   // scanner lines of d_list
constexpr int kListLineWords = 8;     // one 64-byte line
constexpr int kListLines = 1 + kTopM; // line 0: the M candidate words, lines 1..M: row values of candidate m
constexpr int kMaxDomLevels = 8;      // topology levels of all Topology CRs together (rows keep one domain id per level)
constexpr int kDomBuckets = 4096;     // preferred-level domains that can carry a node score at a time

constexpr int kActiveUsed = KAI_POD_ALLOCATED | KAI_POD_PIPELINED | KAI_POD_BINDING | KAI_POD_BOUND |
                            KAI_POD_RUNNING | KAI_POD_RELEASING;
constexpr int kActiveAllocated =
    KAI_POD_ALLOCATED | KAI_POD_PIPELINED | KAI_POD_BINDING | KAI_POD_BOUND | KAI_POD_RUNNING;
constexpr int kAlive = kActiveAllocated | KAI_POD_PENDING | KAI_POD_GATED;
constexpr int kAllocatedStatuses = KAI_POD_ALLOCATED | KAI_POD_BOUND | KAI_POD_BINDING | KAI_POD_RUNNING;

// ---------------------------------------------------------------------------------------------
// shared by the kernels and the host sequencer
// ---------------------------------------------------------------------------------------------
#define KAI_HD __host__ __device__
// full unrolling in device code of shared functions (the host compiler does not know the pragma)
#ifdef __CUDA_ARCH__
#define KAI_UNROLL _Pragma("unroll")
#else
#define KAI_UNROLL
#endif

// IEEE binary64 without contraction on both sides
KAI_HD inline double kadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;  // host translation unit is built with -ffp-contract=off
#endif
}
KAI_HD inline double ksub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
KAI_HD inline double kmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
KAI_HD inline double kdiv(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
KAI_HD inline unsigned long long kbits(double x) {
  unsigned long long u;
  memcpy(&u, &x, 8);
  return u;
}
// Sort key of a list candidate's score: ascending key = descending score for every non-NaN double, negatives and
// +-inf included, and -0.0 gets the key of +0.0 (they compare equal, so the name rank decides between them).  Negative
// scores keep their bits (a larger magnitude sorts later); non-negative ones flip the 63 value bits, which keeps their
// relative order and clears the top bit.  Every key is at most 0xfff0000000000000 (-inf), below ~0ull (an empty slot).
KAI_HD inline unsigned long long list_key(double x) {
  unsigned long long u = kbits(x);
  if (u == 0x8000000000000000ull) u = 0;  // -0.0
  return (u >> 63) ? u : u ^ 0x7fffffffffffffffull;
}
KAI_HD inline double requestable_share(double max_allowed, double request) {
  if (max_allowed == KAI_UNLIMITED) return request;
  return fmin(max_allowed, request);
}
// resource_share.go:51-61
KAI_HD inline double allocatable_share(double deserved, double fair, double max_allowed) {
  if (deserved == KAI_UNLIMITED) return max_allowed;
  double a = fmax(deserved, fair);
  if (max_allowed != KAI_UNLIMITED) a = fmin(max_allowed, a);
  return a;
}

KAI_HD inline unsigned long long make_job_key(int priority, int cls, int order_rank) {
  unsigned long long pinv = (unsigned long long)(unsigned int)(0x40000000 - priority) & 0x7fffffffull;
  return (pinv << 33) | ((unsigned long long)cls << 31) | (unsigned long long)(order_rank & 0x7fffffff);
}

struct Track {  // global min/max of NonAllocated(res) over nodes with Allocatable(res) != 0 (pack.go:66-86)
  double mn, mx;
  int cnt_mn, cnt_mx;
  int dirty;
};
// Merge of two partial binpack extremes (pack.go:66-86) given as (value, number of rows at it): (v, cnt) into (m, c).
// `lower` merges minima, else maxima; a side without rows (count 0) carries no value.
KAI_HD inline void merge_extreme(double &m, long long &c, double v, long long cnt, bool lower) {
  if (cnt <= 0) return;
  if (c == 0 || (lower ? v < m : v > m)) {
    m = v;
    c = cnt;
  } else if (v == m) {
    c += cnt;
  }
}
// tracker event bits per resource (gpu bits 0-2, cpu bits 3-5)
enum { WF_B_EQ_MX = 1, WF_A_EQ_MN = 2, WF_A_LT_MN = 4 };
KAI_HD inline uint32_t track_flags(const Track &t, double b, double a) {
  uint32_t f = 0;
  if (b == t.mx) f |= WF_B_EQ_MX;
  if (a < t.mn)
    f |= WF_A_LT_MN;
  else if (a == t.mn)
    f |= WF_A_EQ_MN;
  return f;
}

constexpr uint32_t kTileDom = 1u << 29;  // tile flag bits 29, 28, 27, 26: row belongs to the domain selected in slot 0..3
constexpr int kDomSlots = 4;             // nesting depth of SubGroupSet / PodSet constraints the scanners can intersect
// XB_RESTRICT_DOM sweeps carry the number of active slots in xbits bits 8..10: a row must sit in all of them
KAI_HD inline uint32_t dom_need_mask(unsigned int xbits) {
  const unsigned int n = (xbits >> 8) & 7u;
  uint32_t m = 0;
  for (unsigned int i = 0; i < n && i < (unsigned int)kDomSlots; i++) m |= kTileDom >> i;
  return m;
}

struct Tile {  // node tile of one scanner CTA
  double *I, *L;        // [R][npc]
  double *Agpu, *Acpu;  // [npc]
  double *gpu_count;    // [npc]
  int *rank;            // [npc]
  uint32_t *flags;      // [npc]
  int *node;            // [npc] node index of the row
  int *dom;             // [n_dom_levels][npc] topology domain per level
  int n_dom_levels;
  int npc, count, R;
  // Rows are striped by NAME RANK over the GPUs of the box and over the scanners of a GPU: row j of scanner `my`
  // of shard `shard` is the node of name rank (j * nscan + my) * nshard + shard.  Consecutive ranks land on
  // different scanners, so the global top-K rows of a sweep come from ~K different scanners.
  int nscan, my, nshard, shard;
  int nscan_log2;  // log2(nscan) when nscan is a power of two, else -1
};
KAI_HD inline int tile_row_rank(const Tile &tl, int ln) { return (ln * tl.nscan + tl.my) * tl.nshard + tl.shard; }
KAI_HD inline bool tile_owns(const Tile &tl, unsigned int rank, int &ln) {
  unsigned int q = rank;
  if (tl.nshard != 1) {  // one GPU: every rank is this shard's
    q = rank / (unsigned int)tl.nshard;
    if (rank - q * (unsigned int)tl.nshard != (unsigned int)tl.shard) return false;
  }
  unsigned int j;
  if (tl.nscan_log2 >= 0) {  // scanner count is a power of two (256 by default): no integer division on the device
    j = q >> tl.nscan_log2;
    if ((q & ((1u << tl.nscan_log2) - 1u)) != (unsigned int)tl.my) return false;
  } else {
    j = q / (unsigned int)tl.nscan;
    if (q - j * (unsigned int)tl.nscan != (unsigned int)tl.my) return false;
  }
  ln = (int)j;
  return true;
}

// ---- node mutations (node_info.go:457-551) are queued as deltas for the scanner that owns the node ----
enum { ND_ADD = 0, ND_ADD_PIPELINED = 1, ND_ADD_RELEASING = 2, ND_REM = 3, ND_REM_PIPELINED = 4, ND_REM_RELEASING = 5,
       ND_FEAS_SET = 6, ND_FEAS_CLR = 7 };  // 6, 7: feasible-set membership of the row (no task attached)
// applied by the owning scanner to its tile row (lane r handles resource r) and by the host to its node mirror
KAI_HD inline void apply_delta_row(double &I, double &L, int code, double v) {
  switch (code) {
    case ND_ADD: I = ksub(I, v); break;
    case ND_ADD_PIPELINED: L = ksub(L, v); break;
    case ND_ADD_RELEASING: L = kadd(L, v); I = ksub(I, v); break;
    case ND_REM: I = kadd(I, v); break;
    case ND_REM_PIPELINED: L = kadd(L, v); break;
    case ND_REM_RELEASING: L = ksub(L, v); I = kadd(I, v); break;
  }
}

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

// Mutable state the host sequencer works on.  The "hot" per-queue arrays are its own copy; the cold arrays are the
// session arrays of the host mirror themselves (single copy).
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

// Parameters of k_record and k_merge_cluster for one action.
struct ActionParams {
  DevSnap s;
  kai_config cfg;
  int scanners;              // CTAs of k_record
  int nodes_per_cta;         // node rows per scanner (tile height)
  unsigned long long *xbuf;  // answer slots of the scanners (single row / min-max): [kMaxGrid][8] u64
  unsigned long long *mmbuf; // XB_FUSED_MM exchange inside one launch: [kMaxGrid][8] u64, tagged with the sequence number
  long long *counters;       // [48]: watchdog (24..27) and KAI_PROFILE cycle counts
  // this GPU's reduced single-row / min-max answer line in (shared) host memory: lines [2][ranks][kLineWords], parity by
  // sequence number, this GPU's line of parity 0
  unsigned long long *h_slot, *h_mmslot;
  int spin_log2;             // watchdog: polls before a wait is declared dead
  int topm;                  // scanners answer with their kTopM best rows (0 = single best through the last CTA)
  unsigned long long *d_list;  // [kListScanners][kListLines][kListLineWords]: the scanners' top-M lines
  const int *node_domain;    // [n_dom_levels][N] topology domain of every node per level (-1 = label missing), or null
  int n_dom_levels;
  unsigned char *g_tiles;      // [scanners][g_tile_stride] tiles in the layout of tile_carve
  size_t g_tile_stride, tile_bytes;
  unsigned char *g_scan_state; // [scanners][kScanStateBytes]: preferred level + per-domain score buckets of each scanner
  unsigned int *ticket;        // CTAs that finished the current launch (the last one reduces the answers)
  double *mm_result;           // [4] gpu mn, gpu mx, cpu mn, cpu mx of the last MINMAX launch (read by XB_FUSED_MM sweeps)
  unsigned long long *h_clist; // this GPU's merged candidate list [2][kCListWords] in (shared) host memory
  int fused_in_kernel;         // XB_FUSED_MM sweeps exchange their extremes inside the launch (cooperative launch: all CTAs resident)
};

constexpr int kMergeCap = 1024;                      // candidates k_merge_cluster sorts, one per thread (scanners x kTopM)
constexpr int kCEntryWords = 6;                      // score, meta, Ig, Lg, Ic, Lc
constexpr int kCListWords = 2 + kMergeCap * kCEntryWords;  // header {count | more << 31, sequence number} + entries
// A single-row or min-max answer line in host memory: payload words, then the record's sequence number in the last word,
// written after a system fence (the host waits on that word alone)
constexpr int kLineWords = 8;
constexpr int kScanStateBytes = 16 + kDomBuckets;
constexpr int kMaxDeltaL = kMaxDelta;
enum { DK_LOAD = 6 };  // load the tiles from the session tables (first launch of an action)

// One decision record, passed to k_record by value in the kernel parameter space.
struct LaunchRec {
  unsigned long long dw[kDecWords];
  uint64_t seq;
  int n_delta;
  unsigned int dkey[kMaxDeltaL];    // name rank | code << 28, or an extended entry (bit 31)
  unsigned int dtask[kMaxDeltaL];
  unsigned char dcount[kMaxDeltaL]; // repeat count - 1
};

}  // namespace kai
