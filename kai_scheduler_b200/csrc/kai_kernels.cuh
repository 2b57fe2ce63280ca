// kai_kernels.cuh — sm_90a kernels of the scheduling-cycle engine.
//
//   k_node_totals    Σ node Allocatable over ready nodes          (proportion.go:252-288)  } exact or in the
//   k_queue_usage    per-queue Allocated / Request scatter-add    (proportion.go:347-401)  } oracle's order
//   k_queue_usage_ordered  the oracle's order where k_queue_usage's sums could round      } (DESIGN.md §2)
//   k_fair_share     hierarchical fair-share division per level   (resource_division.go:26-357)
//
// The sweep kernels of an action are in kai_action.cuh.
//
// All arithmetic that feeds a decision is IEEE binary64 with explicit round-to-nearest
// intrinsics (no FMA contraction; the file is also compiled with -fmad=false) in the
// reference's operation order (SURVEY.md Appendix A.2/A.3).
#pragma once
#include <cfloat>
#include <cstdint>

#include "kai_device.cuh"

namespace kai {

// ---------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_relaxed_b128(void *p, unsigned long long lo, unsigned long long hi) {
  asm volatile("{ .reg .b128 q; mov.b128 q, {%1, %2}; st.relaxed.gpu.global.b128 [%0], q; }" ::"l"(p), "l"(lo),
               "l"(hi)
               : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_b128(void *p, unsigned long long lo, unsigned long long hi) {
  asm volatile("{ .reg .b128 q; mov.b128 q, {%1, %2}; st.relaxed.sys.global.b128 [%0], q; }" ::"l"(p), "l"(lo),
               "l"(hi)
               : "memory");
}
__device__ __forceinline__ void ld_relaxed_sys_b128(const void *p, unsigned long long &lo, unsigned long long &hi) {
  asm volatile("{ .reg .b128 q; ld.relaxed.sys.global.b128 q, [%2]; mov.b128 {%0, %1}, q; }"
               : "=l"(lo), "=l"(hi)
               : "l"(p)
               : "memory");
}
__device__ __forceinline__ void ld_relaxed_b128(const void *p, unsigned long long &lo, unsigned long long &hi) {
  asm volatile("{ .reg .b128 q; ld.relaxed.gpu.global.b128 q, [%2]; mov.b128 {%0, %1}, q; }"
               : "=l"(lo), "=l"(hi)
               : "l"(p)
               : "memory");
}

// ---------------------------------------------------------------------------------------------
// Exact-or-ordered rule of the open-session sums (DESIGN.md §2).  The oracle adds in ascending index order.  When every
// summand of a resource is an integer and the sum of their magnitudes is at most 2^53, every partial sum of any subset,
// in any order and association, is an exact integer, so the parallel tree + atomics below give the oracle's bits.
// Otherwise that resource is redone in the oracle's order.
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kExactSat = (1ull << 53) + 1;  // sums of magnitudes saturate here: "above 2^53"
__device__ __forceinline__ void note_summand(double v, int r, unsigned long long &sum, unsigned &inexact) {
  const double a = fabs(v);
  if (v == trunc(v) && a <= 9007199254740992.0)
    sum = min(sum + (unsigned long long)a, kExactSat);
  else
    inexact |= 1u << r;  // fractional, above 2^53, inf or NaN
}
__device__ __forceinline__ bool sums_exact(const volatile OpenSums *os, int which, int r) {
  return !((os->inexact[which] >> r) & 1u) && os->sum_abs[which][r] < kExactSat;
}
// Adds this block's flags and magnitude sums to os.  A block adds at most 256 * kExactSat < 2^62 and at most kExactSat
// per block reaches the global counter, so it cannot wrap below 2048 blocks (the grids are at most 8 per SM).  With
// want_last, returns true in the block that finished last, which then sees every block's sums and flags.
__device__ bool open_sums_publish(OpenSums *os, int which, const unsigned long long *sum, unsigned inexact,
                                  bool want_last) {
  __shared__ unsigned long long ssum[QR];
  __shared__ unsigned sbits;
  __shared__ bool last;
  if (threadIdx.x < QR) ssum[threadIdx.x] = 0;
  if (threadIdx.x == 0) sbits = 0;
  __syncthreads();
  // a warp's 32 sums (each at most kExactSat) first, so that the shared atomics see one add per warp
  for (int r = 0; r < QR; r++) {
    unsigned long long x = sum[r];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0 && x) atomicAdd(&ssum[r], x);
  }
  inexact = __reduce_or_sync(0xffffffffu, inexact);
  if ((threadIdx.x & 31) == 0 && inexact) atomicOr(&sbits, inexact);
  __syncthreads();
  if (threadIdx.x < QR && ssum[threadIdx.x]) atomicAdd(&os->sum_abs[which][threadIdx.x], min(ssum[threadIdx.x], kExactSat));
  if (threadIdx.x == 0 && sbits) atomicOr(&os->inexact[which], sbits);
  if (!want_last) return false;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&os->blocks_done[which], 1u) == gridDim.x - 1;
  __syncthreads();
  if (last) __threadfence();
  return last;
}

// One warp adds n summands in index order, NV sums side by side; lane 0 writes them to out.  The lanes stage a chunk of
// summands in shared memory (their loads are independent and overlap), then lane 0 runs the add chain over the chunk.
// get(k, v) fills v[] with the k-th summands; a summand that does not count stays +0.0, which leaves the sum unchanged:
// a sum started at +0.0 is never -0.0 under round-to-nearest, and x + 0.0 == x for every other x.
constexpr int kOrdChunk = 128;
template <int NV, class F>
__device__ void warp_ordered_sums(int n, F get, double (*buf)[kOrdChunk], double *out) {
  const int lane = threadIdx.x & 31;
  double acc[NV];
  for (int c = 0; c < NV; c++) acc[c] = 0.0;
  for (int base = 0; base < n; base += kOrdChunk) {
    for (int i = lane; i < kOrdChunk; i += 32) {
      double v[NV];
      for (int c = 0; c < NV; c++) v[c] = 0.0;
      if (base + i < n) get(base + i, v);
      for (int c = 0; c < NV; c++) buf[c][i] = v[c];
    }
    __syncwarp();
    if (lane == 0) {
      const int m = min(kOrdChunk, n - base);
      for (int i = 0; i < m; i++)
        for (int c = 0; c < NV; c++) acc[c] = __dadd_rn(acc[c], buf[c][i]);
    }
    __syncwarp();
  }
  if (lane == 0)
    for (int c = 0; c < NV; c++) out[c] = acc[c];
}

// ---------------------------------------------------------------------------------------------
// K_totals: proportion.setTotalResources (proportion.go:252-288)
// ---------------------------------------------------------------------------------------------
__global__ void k_node_totals(DevSnap s) {
  double acc[QR] = {0, 0, 0};
  unsigned long long mag[QR] = {0, 0, 0};
  unsigned inexact = 0;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < s.N; n += gridDim.x * blockDim.x) {
    if (!(s.nflags[n] & KAI_NODE_READY)) continue;
    for (int r = 0; r < QR; r++) {
      double v = s.alloc[(size_t)r * s.N + n];
      if (s.foreign) v = __dsub_rn(v, s.foreign[(size_t)r * s.N + n]);
      acc[r] = __dadd_rn(acc[r], v);
      note_summand(v, r, mag[r], inexact);
    }
  }
  __shared__ double sh[QR][32];
  for (int r = 0; r < QR; r++) {
    double v = acc[r];
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sh[r][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < QR) {
    double v = 0;
    for (int w = 0; w < (blockDim.x + 31) / 32; w++) v = __dadd_rn(v, sh[threadIdx.x][w]);
    atomicAdd(&s.total[threadIdx.x], v);
  }
  if (!open_sums_publish(s.osum, 0, mag, inexact, true)) return;
  // last block: warp r redoes resource r in ascending node index, as the oracle adds
  __shared__ double buf[QR][1][kOrdChunk];
  const int r = threadIdx.x >> 5;
  if (r >= QR || sums_exact(s.osum, 0, r)) return;
  double out;
  warp_ordered_sums<1>(s.N, [&](int n, double *v) {
    if (!(s.nflags[n] & KAI_NODE_READY)) return;
    double x = s.alloc[(size_t)r * s.N + n];
    if (s.foreign) x = __dsub_rn(x, s.foreign[(size_t)r * s.N + n]);
    v[0] = x;
  }, buf[r], &out);
  if ((threadIdx.x & 31) == 0) s.total[r] = out;
}

// ---------------------------------------------------------------------------------------------
// K_usage: proportion.updateQueuesCurrentResourceUsage (proportion.go:347-401)
// ---------------------------------------------------------------------------------------------
__global__ void k_queue_usage(DevSnap s) {
  unsigned long long mag[QR] = {0, 0, 0};
  unsigned inexact = 0;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < s.T; t += gridDim.x * blockDim.x) {
    int st = s.t_status[t];
    bool allocated = (st & kAllocatedStatuses) != 0;
    if (!allocated && st != KAI_POD_PENDING) continue;
    int j = s.t_job[t];
    bool preemptible = (s.j_flags[j] & KAI_JOB_PREEMPTIBLE) != 0;
    if (s.j_queue[j] >= 0)  // every queue sum adds a subset of these summands
      for (int r = 0; r < QR; r++) note_summand(s.t_req[(size_t)t * s.R + r], r, mag[r], inexact);
    for (int q = s.j_queue[j]; q >= 0; q = s.q_parent[q])
      for (int r = 0; r < QR; r++) {
        double v = s.t_req[(size_t)t * s.R + r];
        if (v == 0) continue;
        atomicAdd(&s.q_request[(size_t)r * s.Q + q], v);
        if (allocated) {
          atomicAdd(&s.q_alloc[(size_t)r * s.Q + q], v);
          if (!preemptible) atomicAdd(&s.q_alloc_np[(size_t)r * s.Q + q], v);
        }
      }
  }
  open_sums_publish(s.osum, 1, mag, inexact, false);
}

// Runs after k_queue_usage: one warp per (resource, queue) of a resource whose sums could round redoes that queue's
// Request / Allocated / AllocatedNonPreemptible in the oracle's order (job, podset, task = the caller's task index
// order).  q_tasks lists the tasks under each queue in that order, so the work is O(T * depth) per resource.
__global__ void k_queue_usage_ordered(DevSnap s) {
  __shared__ double buf[8][3][kOrdChunk];
  const int warp = threadIdx.x >> 5;
  const int item = blockIdx.x * (blockDim.x >> 5) + warp;
  if (warp >= 8 || item >= QR * s.Q) return;
  const int r = item / s.Q, q = item % s.Q;
  if (sums_exact(s.osum, 1, r)) return;
  const int *list = s.q_tasks + s.q_task_begin[q];
  double out[3];
  warp_ordered_sums<3>(s.q_task_begin[q + 1] - s.q_task_begin[q], [&](int k, double *v) {
    const int t = list[k];
    const int st = s.t_status[t];
    const bool allocated = (st & kAllocatedStatuses) != 0;
    if (!allocated && st != KAI_POD_PENDING) return;
    const double x = s.t_req[(size_t)t * s.R + r];
    v[0] = x;
    if (allocated) {
      v[1] = x;
      if (!(s.j_flags[s.t_job[t]] & KAI_JOB_PREEMPTIBLE)) v[2] = x;
    }
  }, buf[warp], out);
  if ((threadIdx.x & 31) == 0) {
    s.q_request[(size_t)r * s.Q + q] = out[0];
    s.q_alloc[(size_t)r * s.Q + q] = out[1];
    s.q_alloc_np[(size_t)r * s.Q + q] = out[2];
  }
}

// ---------------------------------------------------------------------------------------------
// K_fairshare: resource_division.SetResourcesShare for every sibling group of one tree level.
// One thread per (group, resource); groups of a level are independent, resources are independent.
// scratch: w [3][Q], rr [3][Q] (NaN = absent)
// ---------------------------------------------------------------------------------------------
struct FsGroup {
  const int *members;
  int n;
};
__device__ __forceinline__ FsGroup fs_group(const DevSnap &s, int parent) {
  FsGroup g;
  if (parent < 0) {
    g.members = s.top_queues;
    g.n = s.n_top;
  } else {
    g.members = s.q_children + s.q_child_begin[parent];
    g.n = s.q_child_begin[parent + 1] - s.q_child_begin[parent];
  }
  return g;
}

__device__ void fs_set_resource_share(const DevSnap &s, FsGroup g, int r, double total, double k, double *w,
                                      double *rr) {
  const size_t ro = (size_t)r * s.Q;
  const double *deserved = s.q_deserved + ro, *limit = s.q_limit + ro, *oqw = s.q_oqw + ro;
  const double *request = s.q_request + ro;
  const double *usage = s.q_usage ? s.q_usage + ro : nullptr;
  double *fair = s.q_fair + ro;
  w += ro;
  rr += ro;
  auto satisfied = [&](int q) {  // resource_division.go:283-290
    if (request[q] <= fair[q]) return true;
    if (limit[q] != KAI_UNLIMITED && limit[q] <= fair[q]) return true;
    return false;
  };
  auto remaining_requested = [&](int q) {  // :317-325
    double requested = requestable_share(limit[q], request[q]);
    if (requested < fair[q]) return 0.0;
    return __dsub_rn(requested, fair[q]);
  };
  // :92-109 setDeservedResource
  double remaining = total;
  for (int i = 0; i < g.n; i++) {
    int q = g.members[i];
    double d = deserved[q];
    if (d == KAI_UNLIMITED) d = total;
    double amount = fmin(d, requestable_share(limit[q], request[q]));
    fair[q] = __dadd_rn(fair[q], amount);
    remaining = __dsub_rn(remaining, amount);
    rr[q] = __longlong_as_double(0x7ff8000000000000LL);
  }
  if (!(remaining > 0)) return;
  // :111-144 divideOverQuotaResource — priorities in descending order (:146-162)
  for (int pass = 0; pass < 2; pass++) {
    long long cur_prio = 0x7fffffffffLL;
    for (;;) {
      long long p = -0x7fffffffffLL;
      bool any = false;
      for (int i = 0; i < g.n; i++) {
        long long qp = s.q_priority[g.members[i]];
        if (qp < cur_prio && (!any || qp > p)) {
          p = qp;
          any = true;
        }
      }
      if (!any) break;
      cur_prio = p;
      if (pass == 0) {
        // :164-222 divideUpToFairShare over the queues of this priority
        for (;;) {
          bool another = false;
          double round_amount = remaining;
          double total_weights = 0;  // :307-315
          for (int i = 0; i < g.n; i++) {
            int q = g.members[i];
            if (s.q_priority[q] != p) continue;
            if (remaining_requested(q) > 0) total_weights = __dadd_rn(total_weights, oqw[q]);
          }
          double wsum = 0.0;
          if (total_weights != 0) {  // :224-251 calcShareWeights
            for (int i = 0; i < g.n; i++) {
              int q = g.members[i];
              if (s.q_priority[q] != p) continue;
              w[q] = 0.0;
              if (satisfied(q)) continue;
              double n_weight = __ddiv_rn(oqw[q], total_weights);
              double n_usage = usage ? usage[q] : 0.0;
              double t = __dsub_rn(n_weight, n_usage);
              double t2 = __dmul_rn(k, t);
              double sw = fmax(0.0, __dadd_rn(n_weight, t2));
              w[q] = sw;
              wsum = __dadd_rn(wsum, sw);
            }
          }
          if (wsum == 0) break;
          for (int i = 0; i < g.n; i++) {
            int q = g.members[i];
            if (s.q_priority[q] != p) continue;
            if (remaining == 0) break;
            if (satisfied(q)) continue;
            double requested = remaining_requested(q);
            if (oqw[q] == 0) continue;
            double nqw = __ddiv_rn(w[q], wsum);
            double fs = __dmul_rn(round_amount, nqw);
            double give = 0;  // :264-281 getResourceToGiveInCurrentRound
            if (requested <= fs) {
              give = requested;
              rr[q] = __longlong_as_double(0x7ff8000000000000LL);
            } else {
              double rf = floor(fs);
              if (rf > 0) give = rf;
              double left = __dsub_rn(fs, give);
              if (left > 0) rr[q] = left;
            }
            if (give == 0) continue;
            fair[q] = __dadd_rn(fair[q], give);
            remaining = __dsub_rn(remaining, give);
            another = another || requested < fs;
          }
          if (!another || remaining == 0) break;
        }
      } else {
        if (remaining <= 0) break;
        // :253-262 divideRemainingResource, order :335-357 (remaining desc, creation asc, uid asc)
        for (;;) {
          if (remaining == 0) break;
          int best = -1;
          for (int i = 0; i < g.n; i++) {
            int q = g.members[i];
            if (s.q_priority[q] != p) continue;
            double a = rr[q];
            if (a != a) continue;
            if (best < 0) {
              best = q;
              continue;
            }
            double b = rr[best];
            bool better;
            if (a > b)
              better = true;
            else if (a < b)
              better = false;
            else if (s.q_creation[q] != s.q_creation[best])
              better = s.q_creation[q] < s.q_creation[best];
            else
              better = s.q_uid_rank[q] < s.q_uid_rank[best];
            if (better) best = q;
          }
          if (best < 0) break;
          rr[best] = __longlong_as_double(0x7ff8000000000000LL);
          double give = fmin(1.0, remaining);
          fair[best] = __dadd_rn(fair[best], give);
          remaining = __dsub_rn(remaining, give);
        }
      }
    }
  }
}

// single CTA; levels separated by __syncthreads (proportion.go:410-423 setFairShareForQueues)
__global__ void k_fair_share(DevSnap s, double k_value, double *w, double *rr) {
  for (int lvl = 0; lvl < s.n_levels; lvl++) {
    int g0 = s.level_group_begin[lvl], g1 = s.level_group_begin[lvl + 1];
    int n_items = (g1 - g0) * QR;
    for (int it = threadIdx.x; it < n_items; it += blockDim.x) {
      int parent = s.level_groups[g0 + it / QR];
      int r = it % QR;
      double total = parent < 0 ? s.total[r] : s.q_fair[(size_t)r * s.Q + parent];
      fs_set_resource_share(s, fs_group(s, parent), r, total, k_value, w, rr);
    }
    __syncthreads();
  }
  // GetAllocatableShare per queue (resource_share.go:51-61): static for the rest of the cycle
  for (int i = threadIdx.x; i < QR * s.Q; i += blockDim.x)
    s.q_allocatable[i] = allocatable_share(s.q_deserved[i], s.q_fair[i], s.q_limit[i]);
}

}  // namespace kai
