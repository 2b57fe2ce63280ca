// kai_action.cuh — the action kernels and the two prepare kernels.
//
//   k_prep_jobs      per job: podset status counters, readiness, JobOrderFn sort key, cached
//                    GetTasksToAllocateInitResource, "fresh uniform gang" flag                (grid-parallel)
//   k_prep_queues    per leaf queue: eligible jobs in JobOrderFn order                        (CTA per queue)
//   k_record         ONE decision record of the host sequencer per launch, 256 scanners x 128 threads.  Every scanner
//                    owns a stripe of node rows (tile, resident in global memory / L2 between launches, staged in
//                    shared memory for the sweep), applies the node deltas addressed to it, evaluates fit + score of
//                    its rows and answers: top-M candidates (lists), or one slot reduced by the last CTA to finish.
//   k_merge_cluster  sorts the scanners' candidates, cuts the list where an unseen row could be better and streams it
//                    to host memory — the next launch on the stream after a list sweep.
//
// Exactness notes
//   * FittingNode + NodeOrderFn + sortNodesByScore (framework/session.go:201-264,466-485) are evaluated as
//     "argmax over fitting nodes of (score desc, name-rank asc)" with the reference's f64 operation order.
//   * binpack min/max (pack.go:66-86) are tracked incrementally with counts of nodes at the extremes; any
//     event that could change an extreme without being observable marks the tracker dirty and forces a
//     min/max exchange before the next sweep that needs it.
//   * same-node batching: after a sweep picked node n for a pod, the owner of n also reports for how many
//     further pods with the SAME request/flags node n provably stays the argmax (its score does not drop
//     below the winning score, it still fits in the same mode, min/max stay put).  Those pods are placed
//     without a sweep.  DESIGN.md §5 has the argument.
#pragma once
#include <cfloat>
#include <cstdint>

#include <cooperative_groups.h>

#include "kai_device.cuh"
#include "kai_kernels.cuh"
#include "kai_seq.cuh"

namespace kai {

// ---------------------------------------------------------------------------------------------
// prepare kernels
// ---------------------------------------------------------------------------------------------
__global__ void k_prep_jobs(DevSnap s, int filter_non_pending, int filter_unready) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < s.J; j += gridDim.x * blockDim.x) {
    bool ready = true, below = false, exactly = true;
    int pending = 0;
    for (int ps = s.j_ps_begin[j]; ps < s.j_ps_begin[j + 1]; ps++) {
      int act = 0, pend = 0, pipe = 0, alive = 0, gated = 0;
      for (int i = s.ps_task_begin[ps]; i < s.ps_task_begin[ps + 1]; i++) {
        int st = s.t_status[i];  // tasks of a podset are contiguous
        if (st & kActiveAllocated) act++;
        if (st == KAI_POD_PENDING) pend++;
        if (st == KAI_POD_PIPELINED) pipe++;
        if (st & kAlive) alive++;
        if (st & KAI_POD_GATED) gated++;
      }
      s.ps_cnt0[ps] = act;
      s.ps_cnt0[s.S + ps] = pend;
      s.ps_cnt0[2 * s.S + ps] = pipe;
      int m = s.ps_min[ps];
      if (alive - gated < m) ready = false;  // podset.go:114-120
      pending += pend;
      if (act < m) below = true;  // elastic.go:50-63
      if (act > m) exactly = false;
    }
    int cls = below ? 0 : (exactly ? 1 : 2);
    int q = s.j_queue[j];
    bool eligible = (!filter_unready || ready) && (!filter_non_pending || pending > 0) && q >= 0 &&
                    s.q_nchildren[q] == 0;  // input_jobs.go:24-63
    s.j_key0[j] = eligible ? make_job_key(s.j_priority[j], cls, s.j_order_rank[j]) : kKeyNone;
    // GetTasksToAllocateInitResource(job, isRealAllocation=false) (allocation_info.go:87-113) for the common
    // single-podset job; other jobs are evaluated lazily by the sequencer.  Tasks of a podset are stored in
    // TaskOrderFn order (the host renumbers them), so "the first k that should allocate" is a linear scan.
    s.j_req_valid[j] = 0;
    JobRec rec;
    rec.req0[0] = rec.req0[1] = rec.req0[2] = 0;
    rec.n_tta = -1;
    rec.ps0 = s.j_ps_begin[j];
    rec.n_podsets = s.j_ps_begin[j + 1] - s.j_ps_begin[j];
    rec.tb = rec.n_podsets > 0 ? s.ps_task_begin[rec.ps0] : 0;
    rec.cnt[0] = rec.cnt[1] = rec.cnt[2] = 0;
    rec.pad[0] = rec.pad[1] = rec.pad[2] = 0;
    if (rec.n_podsets == 1) {
      int ps = rec.ps0;
      int act = s.ps_cnt0[ps], m = s.ps_min[ps];
      rec.cnt[0] = act;
      rec.cnt[1] = s.ps_cnt0[s.S + ps];
      rec.cnt[2] = s.ps_cnt0[2 * s.S + ps];
      int max_tasks = act >= m ? 1 : m - act;
      double sum[QR] = {0, 0, 0};
      int taken = 0;
      bool prefix = true;  // the selected tasks are exactly the first `taken` tasks and all are Pending
      for (int t = s.ps_task_begin[ps]; t < s.ps_task_begin[ps + 1] && taken < max_tasks; t++) {
        int st = s.t_status[t];
        if (!(st == KAI_POD_PENDING || (st == KAI_POD_RELEASING && s.t_virtual[t]))) {
          prefix = false;
          continue;
        }
        if (st != KAI_POD_PENDING) prefix = false;
        for (int r = 0; r < QR; r++) sum[r] = __dadd_rn(sum[r], s.t_req[(size_t)t * s.R + r]);
        taken++;
      }
      for (int r = 0; r < QR; r++) {
        s.j_req[(size_t)j * QR + r] = sum[r];
        rec.req0[r] = sum[r];
      }
      s.j_req_valid[j] = 1;
      if (prefix && act == 0 && rec.cnt[2] == 0) {
        rec.n_tta = taken;
        // pad[0]: the selected tasks are interchangeable for the sweep (bit-identical request, nominated node, predicate
        // class): the host sequencer may defer their per-task bookkeeping until the gang is complete
        bool uniform = taken >= 1;
        const int t0 = rec.tb;
        for (int t = t0 + 1; t < t0 + taken && uniform; t++) {
          for (int r = 0; r < s.R; r++)
            if (__double_as_longlong(s.t_req[(size_t)t * s.R + r]) != __double_as_longlong(s.t_req[(size_t)t0 * s.R + r])) uniform = false;
          if (s.t_nominated && s.t_nominated[t] != s.t_nominated[t0]) uniform = false;
          if (s.t_pred_class && s.t_pred_class[t] != s.t_pred_class[t0]) uniform = false;
        }
        rec.pad[0] = uniform ? 1 : 0;
      }
    }
    s.jrec[j] = rec;
  }
}

// One CTA per leaf queue: parallel compaction of the eligible jobs (block scan), then a parallel check that
// the compacted run is already in JobOrderFn key order (host order is (priority desc, creation, uid); only
// differing elastic classes inside one priority can break it); if not, thread 0 insertion-sorts the run.
__global__ void k_prep_queues(DevSnap s) {
  __shared__ int warp_tot[32];
  __shared__ int base, unsorted;
  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int b = s.q_job_begin[q], e = s.q_job_begin[q + 1];
  int *out = s.leaf_sorted + b;
  if (tid == 0) {
    base = 0;
    unsorted = 0;
  }
  __syncthreads();
  for (int k0 = b; k0 < e; k0 += blockDim.x) {
    int k = k0 + tid;
    int job = k < e ? s.q_jobs_sorted[k] : -1;
    bool el = job >= 0 && s.j_key0[job] != kKeyNone;
    unsigned int m = __ballot_sync(0xffffffffu, el);
    int pre = __popc(m & ((1u << lane) - 1));
    if (lane == 0) warp_tot[warp] = __popc(m);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; w++) off += warp_tot[w];
    if (el) out[off + pre] = job;
    __syncthreads();
    if (tid == 0) {
      int t = 0;
      for (int w = 0; w < nw; w++) t += warp_tot[w];
      base += t;
    }
    __syncthreads();
  }
  const int n = base;
  for (int i = tid + 1; i < n; i += blockDim.x)
    if (s.j_key0[out[i]] < s.j_key0[out[i - 1]]) unsorted = 1;
  __syncthreads();
  if (tid == 0) {
    if (unsorted) {
      for (int i = 1; i < n; i++) {
        int job = out[i];
        unsigned long long key = s.j_key0[job];
        int p = i;
        while (p > 0 && key < s.j_key0[out[p - 1]]) {
          out[p] = out[p - 1];
          p--;
        }
        out[p] = job;
      }
    }
    s.leaf_count[q] = n;
  }
}

// =============================================================================================
// cooperative pieces (all threads of the CTA)
// =============================================================================================
struct Cand {
  double score;
  uint32_t rank;
  int ln;
};
// better / binpack_score / row_fits / row_score / node_key / repeat_row are compiled for the host too: the solver answers
// small restricted sweeps from its node mirror with the very operations the scanners run (kadd & co. are IEEE binary64
// without contraction on both sides)
KAI_HD __forceinline__ bool better(double sa, uint32_t ra, double sb, uint32_t rb) {
  if (ra == kRankNone) return false;
  if (rb == kRankNone) return true;
  return sa > sb || (sa == sb && ra < rb);
}

// pack.go:45-64
KAI_HD __forceinline__ double binpack_score(double mn, double mx, double cur, double overall) {
  if (overall == 0) return 0.0;
  if (mx == 0) return 0.0;
  if (mn == mx) return 9.0;
  double t1 = ksub(cur, mn);
  double t2 = ksub(mx, mn);
  double t3 = kdiv(t1, t2);
  double t4 = ksub(1.0, t3);
  return kmul(9.0, t4);
}

// The rules below take a node row as Idle/Releasing vectors with resource r at [r * stride].  They only ever index it
// with constants after unrolling, so a row held in registers (stride 1) stays in registers.
//
// FittingNode (session.go:201-232) of request rq[R]: returns whether the row fits on Idle + Releasing; fit_i = fits on
// Idle alone.
KAI_HD __forceinline__ bool row_fits(const double *rq, int R, const double *I, const double *L, int stride, bool &fit_i) {
  bool fit_ri = true;
  fit_i = true;
  KAI_UNROLL
  for (int r = 0; r < KAI_MAX_RES; r++) {
    if (r >= R) break;
    double i = I[r * stride];
    double avail = kadd(i, L[r * stride]);
    if (r >= 3) {
      if (rq[r] != 0 && rq[r] > avail) fit_ri = false;
      if (rq[r] != 0 && rq[r] > i) fit_i = false;
    } else {
      if (rq[r] > avail) fit_ri = false;
      if (rq[r] > i) fit_i = false;
    }
  }
  return fit_ri;
}

// NodeOrderFn sum (session_plugins.go:427-437) of node n's row, in the reference's operation order
KAI_HD __forceinline__ double row_score(const Decision &d, const double *I, const double *L, int stride, double a_gpu,
                                        double a_cpu, double gpu_count, uint32_t nflags, int n, bool fit_i) {
  double score = 0.0;
  score = kadd(score, (d.best_effort || fit_i) ? 100.0 : 0.0);  // nodeavailability.go:29-40
  score = kadd(score, 0.0);                                   // gpusharingorder (whole GPUs)
  bool cpu_only_node = !(nflags & KAI_NODE_NOT_CPU_ONLY) && a_gpu <= 0;
  score = kadd(score, (!d.gpu_task && cpu_only_node) ? 10.0 : 0.0);  // resourcetype.go:29-41
  score = kadd(score, (d.nominated == n) ? 1000000.0 : 0.0);        // nominatednode.go:29-41
  const bool gpu = d.res == KAI_RES_GPU;  // the scored resource is GPU or CPU
  double cur = gpu ? kadd(I[KAI_RES_GPU * stride], L[KAI_RES_GPU * stride]) : kadd(I[KAI_RES_CPU * stride], L[KAI_RES_CPU * stride]);
  double overall = gpu ? a_gpu : a_cpu;
  double place;
  if (d.strategy == KAI_PLACEMENT_BINPACK) {
    place = binpack_score(d.mn, d.mx, cur, overall);
  } else {  // spread.go:16-36
    double cnt = gpu ? (double)(long long)gpu_count : overall;
    place = cnt == 0 ? 0.0 : kdiv(cur, cnt);
  }
  return kadd(score, place);
}

// FittingNode + NodeOrderFn of node n's row.  Returns false if the node does not fit; fit_i = fits on Idle alone.
KAI_HD __forceinline__ bool node_key(const Decision &d, int R, const double *I, const double *L, int stride,
                                     double a_gpu, double a_cpu, double gpu_count, uint32_t nflags, int n,
                                     double &score, bool &fit_i) {
  if (!row_fits(d.req, R, I, L, stride, fit_i)) return false;
  score = row_score(d, I, L, stride, a_gpu, a_cpu, gpu_count, nflags, n, fit_i);
  return true;
}

// Same-node repeats (DESIGN.md §5): row ln of the tile after k placements of d's request, in registers.  The mode is
// decided on the row before any placement (common/allocate.go:165-174); the placements subtract the request in order,
// with the f64 operations of the sequential application (node_info.go:457-493).  Returns whether placement k may repeat
// the winning placement: the row still fits (`fits`), in the same mode, and its score plus the row's topology term
// `topo` is at least the winning score `win`, so node ln stays the argmax.
KAI_HD __forceinline__ bool repeat_row(const Tile &tl, const Decision &d, int ln, int k, double win, double topo,
                                       double (&I)[KAI_MAX_RES], double (&L)[KAI_MAX_RES], bool &to_idle, bool &fits) {
  const int R = tl.R;
  double rq[KAI_MAX_RES];
  KAI_UNROLL
  for (int r = 0; r < KAI_MAX_RES; r++) {
    I[r] = r < R ? tl.I[r * tl.npc + ln] : 0.0;
    L[r] = r < R ? tl.L[r * tl.npc + ln] : 0.0;
    rq[r] = r < R ? d.req[r] : 0.0;
  }
  bool fit_i;
  row_fits(rq, R, I, L, 1, fit_i);
  to_idle = !d.pipeline_only && (d.best_effort || fit_i);
  for (int j = 0; j < k; j++) {
    KAI_UNROLL
    for (int r = 0; r < KAI_MAX_RES; r++) {
      if (to_idle)
        I[r] = ksub(I[r], rq[r]);  // rq[r] = 0 beyond R: exact no-op
      else
        L[r] = ksub(L[r], rq[r]);
    }
  }
  fits = row_fits(rq, R, I, L, 1, fit_i);
  if (!fits) return false;
  const double sc = row_score(d, I, L, 1, tl.Agpu[ln], tl.Acpu[ln], tl.gpu_count[ln], tl.flags[ln], tl.node[ln], fit_i);
  return (!d.pipeline_only && (d.best_effort || fit_i)) == to_idle && kadd(sc, topo) >= win;
}

// The sweeps' row set: the restricted feasible set and the selected topology domains
__device__ __forceinline__ bool in_row_set(const Tile &tl, int ln, bool restricted, int xbits) {
  if (restricted && !(tl.flags[ln] & kTileFeas)) return false;
  const uint32_t need = dom_need_mask((unsigned int)xbits);
  return !(xbits & XB_RESTRICT_DOM) || (tl.flags[ln] & need) == need;
}

// argmax on (score desc, name rank asc) over the lanes of a warp: the winner on lane 0
__device__ __forceinline__ Cand warp_argmax(Cand c) {
  for (int o = 16; o > 0; o >>= 1) {
    Cand x;
    x.score = __shfl_down_sync(0xffffffffu, c.score, o);
    x.rank = __shfl_down_sync(0xffffffffu, c.rank, o);
    x.ln = __shfl_down_sync(0xffffffffu, c.ln, o);
    if (better(x.score, x.rank, c.score, c.rank)) c = x;
  }
  return c;
}

// The sweep over this CTA's tile followed by the block argmax on (score desc, name rank asc).  key(ln, score) is the rule
// of the sweep: false when row ln is not a candidate, else its score.  Candidates in excl[0, n_excl) are counted but not
// taken; fit_count (if set) receives the number of candidates.
template <class Key>
__device__ Cand scan_tile(const Tile &tl, Key key, Cand *sh_warp, const int *excl, int n_excl, int *fit_count) {
  Cand best = {-1.0, kRankNone, -1};
  int n_fit = 0;
  for (int ln = threadIdx.x; ln < tl.count; ln += blockDim.x) {
    double score;
    if (!key(ln, score)) continue;
    n_fit++;
    bool skip = false;
    for (int x = 0; x < n_excl; x++)
      if (excl[x] == ln) skip = true;
    if (skip) continue;
    uint32_t rk = (uint32_t)tl.rank[ln];
    if (better(score, rk, best.score, best.rank)) best = {score, rk, ln};
  }
  if (fit_count) {
    int w = __reduce_add_sync(0xffffffffu, n_fit);
    if ((threadIdx.x & 31) == 0 && w) atomicAdd(fit_count, w);
  }
  best = warp_argmax(best);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh_warp[warp] = best;
  __syncthreads();
  if (warp == 0) {
    Cand c = {-1.0, kRankNone, -1};
    if (lane < (int)(blockDim.x >> 5)) c = sh_warp[lane];
    best = warp_argmax(c);
  }
  return best;  // valid on thread 0
}

// The kTopM best candidates of this CTA in key order into cands (a missing one has rank kRankNone; excl lists their rows),
// and the number of candidates into *fit_count
template <class Key>
__device__ void scan_top_m(const Tile &tl, Key key, Cand *sh_warp, int *excl, Cand *cands, int *fit_count) {
  if (threadIdx.x == 0) *fit_count = 0;
  __syncthreads();
  for (int m = 0; m < kTopM; m++) {
    Cand c = scan_tile(tl, key, sh_warp, excl, m, m == 0 ? fit_count : nullptr);
    if (threadIdx.x == 0) {
      cands[m] = c;
      excl[m] = c.ln;
    }
    __syncthreads();
  }
}

// pack.go:66-86 over this CTA's rows of the row set (the predicate mask does not apply): min and max of Idle + Releasing
// of GPU (k = 0) and CPU (k = 1) over the rows whose Allocatable of that resource is not 0, folded over the block
// through sh_d (4 per warp).  Every thread returns the CTA's extremes.
__device__ void tile_extremes(const Tile &tl, bool restricted, int xbits, double *sh_d, double (&mn)[2], double (&mx)[2]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  mn[0] = mn[1] = DBL_MAX;
  mx[0] = mx[1] = 0.0;
  for (int ln = threadIdx.x; ln < tl.count; ln += blockDim.x) {
    if (!in_row_set(tl, ln, restricted, xbits)) continue;
    for (int k = 0; k < 2; k++) {
      int res = k == 0 ? KAI_RES_GPU : KAI_RES_CPU;
      double overall = k == 0 ? tl.Agpu[ln] : tl.Acpu[ln];
      if (overall == 0) continue;
      double cur = __dadd_rn(tl.I[res * tl.npc + ln], tl.L[res * tl.npc + ln]);
      if (cur < mn[k]) mn[k] = cur;
      if (cur > mx[k]) mx[k] = cur;
    }
  }
  for (int k = 0; k < 2; k++)
    for (int o = 16; o > 0; o >>= 1) {
      mn[k] = fmin(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
      mx[k] = fmax(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
    }
  if (lane == 0) {
    sh_d[warp * 4 + 0] = mn[0];
    sh_d[warp * 4 + 1] = mx[0];
    sh_d[warp * 4 + 2] = mn[1];
    sh_d[warp * 4 + 3] = mx[1];
  }
  __syncthreads();
  for (int k = 0; k < 2; k++) {
    mn[k] = DBL_MAX;
    mx[k] = 0.0;
    for (int w = 0; w < nw; w++) {
      mn[k] = fmin(mn[k], sh_d[w * 4 + 2 * k]);
      mx[k] = fmax(mx[k], sh_d[w * 4 + 2 * k + 1]);
    }
  }
}

// answer slot of a scanner in xbuf (8 x u64), read by the last CTA of the same launch after the ticket:
//   single row {score bits, [flags:8][repeat:8][rank:24]} {cur_a gpu bits, cur_a cpu bits} {repeat tracker-event bits, -}
//   min-max    {gpu min, count} {gpu max, count} {cpu min, count} {cpu max, count}
constexpr int kSlotWords = 8;

// candidate of this CTA -> slot words, including the same-node repeat analysis (lane 0 of warp 0)
// Executed by ALL lanes of warp 0 of a scanner.  Lane i evaluates "placement i" on the winning node row
// (i = 0 is the swept placement, i >= 1 are candidate repeats on the same node); lane 0 then walks the
// placements in order to simulate the min/max trackers and decides how many repeats it can vouch for.
__device__ void publish_candidate(const Track *trk, const Tile &tl, const Decision &d, Cand local,
                                  unsigned long long *slot, int batching) {
  const int lane = threadIdx.x & 31;
  local.score = __shfl_sync(0xffffffffu, local.score, 0);
  local.rank = __shfl_sync(0xffffffffu, local.rank, 0);
  local.ln = __shfl_sync(0xffffffffu, local.ln, 0);
  uint32_t flags = 0, repeat = 0;
  double a_gpu = 0, a_cpu = 0;
  unsigned long long rep_flags = 0;
  if (local.rank != kRankNone) {  // warp-uniform
    const int ln = local.ln;
    double I[KAI_MAX_RES], L[KAI_MAX_RES];
    bool to_idle, fits;
    // topology term 0: the repeat's score without it against the swept score with it finds fewer repeats, never a wrong one
    bool ok = repeat_row(tl, d, ln, lane <= kMaxRepeat ? lane : kMaxRepeat, local.score, 0.0, I, L, to_idle, fits);
    const double ag = tl.Agpu[ln], ac = tl.Acpu[ln];
    double b2[2] = {0, 0}, a2[2] = {0, 0};
    int has[2] = {0, 0};
    {
      const double Ig = I[KAI_RES_GPU], Lg = L[KAI_RES_GPU], Ic = I[KAI_RES_CPU], Lc = L[KAI_RES_CPU];
      const double rg = d.req[KAI_RES_GPU], rc = d.req[KAI_RES_CPU];
      if (ag != 0 && rg != 0) {
        has[0] = 1;
        b2[0] = __dadd_rn(Ig, Lg);
        a2[0] = to_idle ? __dadd_rn(__dsub_rn(Ig, rg), Lg) : __dadd_rn(Ig, __dsub_rn(Lg, rg));
      }
      if (ac != 0 && rc != 0) {
        has[1] = 1;
        b2[1] = __dadd_rn(Ic, Lc);
        a2[1] = to_idle ? __dadd_rn(__dsub_rn(Ic, rc), Lc) : __dadd_rn(Ic, __dsub_rn(Lc, rc));
      }
    }
    // Tracker events of placement `lane`.  Within a batch min/max of both resources are constant (the batch
    // ends before any placement that would move them), so every lane can evaluate its events against the
    // trackers of the record; only the "last node leaves the max" rule needs a prefix count.
    uint32_t f6 = 0;
    for (int k = 0; k < 2; k++) {
      if (!has[k] || trk[k].dirty) continue;
      f6 |= track_flags(trk[k], b2[k], a2[k]) << (3 * k);
    }
    if (lane > kMaxRepeat) {
      ok = false;
      f6 = 0;
    }
    const int sk = d.res == KAI_RES_GPU ? 0 : 1;  // scored resource
    const bool tracked = d.strategy == KAI_PLACEMENT_BINPACK && !trk[sk].dirty;
    const uint32_t lt_any = (f6 & WF_A_LT_MN) | ((f6 >> 3) & WF_A_LT_MN);
    const uint32_t eqmx_s = (f6 >> (3 * sk)) & WF_B_EQ_MX;
    const unsigned ok_mask = __ballot_sync(0xffffffffu, ok);
    const unsigned lt_mask = __ballot_sync(0xffffffffu, lt_any != 0);
    const unsigned eq_mask = __ballot_sync(0xffffffffu, eqmx_s != 0);
    // placement j "stops" the batch after itself if it moves min/max of the scored resource or dirties it
    const int n_eq_before = __popc(eq_mask & ((1u << lane) - 1));
    const bool lt_s = ((f6 >> (3 * sk)) & WF_A_LT_MN) != 0;
    const bool stops = tracked && (lt_s || (eqmx_s && n_eq_before + 1 >= trk[sk].cnt_mx));
    const unsigned stop_mask = __ballot_sync(0xffffffffu, stops);
    // repeat i (>= 1) is usable iff ok_i, it establishes no new minimum, and no placement before it stopped
    int rep_n = 0;
    if (batching) {
      for (int i2 = 1; i2 <= kMaxRepeat; i2++) {
        if (!((ok_mask >> i2) & 1u) || ((lt_mask >> i2) & 1u)) break;
        if (stop_mask & ((1u << i2) - 1)) break;
        rep_n = i2;
      }
    }
    repeat = (uint32_t)rep_n;
    if (to_idle) flags |= SLOT_TO_IDLE;
    {
      uint32_t f0 = __shfl_sync(0xffffffffu, f6, 0);
      flags |= f0 & 0x3fu;
      a_gpu = __shfl_sync(0xffffffffu, a2[0], 0);
      a_cpu = __shfl_sync(0xffffffffu, a2[1], 0);
      // pack the event bits of repeats 1..repeat: lane i contributes bits [6(i-1), 6i)
      unsigned lo32 = 0, hi32 = 0;
      if (lane >= 1 && lane <= rep_n) {
        unsigned long long w = (unsigned long long)(f6 & 0x3fu) << (6 * (lane - 1));
        lo32 = (unsigned)(w & 0xffffffffu);
        hi32 = (unsigned)(w >> 32);
      }
      lo32 = __reduce_or_sync(0xffffffffu, lo32);
      hi32 = __reduce_or_sync(0xffffffffu, hi32);
      rep_flags = ((unsigned long long)hi32 << 32) | lo32;
    }
    if (repeat) flags |= SLOT_HAS_REPEAT;
  }
  if (lane != 0) return;
  st_relaxed_b128(slot + 2, (unsigned long long)__double_as_longlong(a_gpu), (unsigned long long)__double_as_longlong(a_cpu));
  if (repeat) st_relaxed_b128(slot + 4, rep_flags, 0ull);
  unsigned long long meta = ((unsigned long long)(flags & 0xffu) << 32) | ((unsigned long long)(repeat & 0xffu) << 24) |
                            (unsigned long long)(local.rank & 0xffffffu);
  st_relaxed_b128(slot, (unsigned long long)__double_as_longlong(local.score), meta);
}


// ---------------------------------------------------------------------------------------------
// top-M answer.  Warp w analyses candidate w: how many further identical pods the row can
// take while staying at or above its own winning score in the same mode (repeat), and whether it is exhausted
// afterwards (does not fit any more).  The host merges the lists of all scanners, simulates the min/max trackers
// itself from the row values (same f64 operations) and consumes the list in key order (DESIGN.md §5).
// ---------------------------------------------------------------------------------------------
enum { LF_TO_IDLE = 1, LF_EXHAUSTED = 2, LF_MORE = 4, LF_HAS_GPU = 8, LF_HAS_CPU = 16 };
__device__ void publish_list_candidate(const Tile &tl, const Decision &d, Cand c, bool more, unsigned long long *line0_word,
                                       unsigned long long *payload_line, double topo_term) {
  const int lane = threadIdx.x & 31;
  uint32_t flags = more ? LF_MORE : 0u, repeat = 0;
  double Ig0 = 0, Lg0 = 0, Ic0 = 0, Lc0 = 0;
  if (c.rank != kRankNone) {  // warp-uniform
    const int ln = c.ln;
    Ig0 = tl.I[KAI_RES_GPU * tl.npc + ln];
    Lg0 = tl.L[KAI_RES_GPU * tl.npc + ln];
    Ic0 = tl.I[KAI_RES_CPU * tl.npc + ln];
    Lc0 = tl.L[KAI_RES_CPU * tl.npc + ln];
    if (tl.Agpu[ln] != 0 && d.req[KAI_RES_GPU] != 0) flags |= LF_HAS_GPU;
    if (tl.Acpu[ln] != 0 && d.req[KAI_RES_CPU] != 0) flags |= LF_HAS_CPU;
    double I[KAI_MAX_RES], L[KAI_MAX_RES];
    bool to_idle, fits;
    // the row's topology score is the same for every repeat
    const bool ok = repeat_row(tl, d, ln, lane <= kMaxRepeat + 1 ? lane : kMaxRepeat + 1, c.score, topo_term, I, L, to_idle, fits);
    if (to_idle) flags |= LF_TO_IDLE;
    const unsigned ok_mask = __ballot_sync(0xffffffffu, ok);
    const unsigned fit_mask = __ballot_sync(0xffffffffu, fits);
    int r_n = 0;
    for (int i2 = 1; i2 <= kMaxRepeat; i2++) {
      if (!((ok_mask >> i2) & 1u)) break;
      r_n = i2;
    }
    repeat = (uint32_t)r_n;
    if (!((fit_mask >> (r_n + 1)) & 1u)) flags |= LF_EXHAUSTED;  // after 1 + repeat placements the row no longer fits
  }
  if (lane == 0) {
    st_relaxed_sys_b128(payload_line + 0, (unsigned long long)__double_as_longlong(Ig0), (unsigned long long)__double_as_longlong(Lg0));
    st_relaxed_sys_b128(payload_line + 2, (unsigned long long)__double_as_longlong(Ic0), (unsigned long long)__double_as_longlong(Lc0));
    unsigned long long hi = ((unsigned long long)(flags & 0xffu) << 32) | ((unsigned long long)(repeat & 0xffu) << 24) |
                            (unsigned long long)(c.rank & 0xffffffu);
    st_relaxed_sys_b128(line0_word, (unsigned long long)__double_as_longlong(c.score), hi);
  }
}

// =============================================================================================
// device-side exchange inside one launch
// =============================================================================================
// Watchdog for the spin wait of the XB_FUSED_MM exchange: a wait that does not complete within ~2^22 polls records (code, seq, who)
// in counters[24..27], raises the abort flag and lets every waiter fall through so that the kernel ends
// and the host reports KAI_ERR_CUDA instead of hanging the GPU.
struct Spin {
  unsigned int n = 0;
  __device__ __forceinline__ bool expired(const ActionParams &p, int code, unsigned long long seq, int who) {
    if ((++n & 0x3ffu) != 0) return false;
    volatile long long *c = p.counters;
    if (c[24] != 0) return true;
    if (n >= (1u << p.spin_log2)) {
      if (atomicCAS((unsigned long long *)&p.counters[24], 0ull, (unsigned long long)code) == 0ull) {
        c[25] = seq;
        c[26] = who;
        c[27] = blockIdx.x;
      }
      return true;
    }
    return false;
  }
};


// =============================================================================================
// scanner CTA
// =============================================================================================
// the arrays of a tile inside one contiguous block (the scanner's block of g_tiles, or its copy in shared memory that a
// sweep reads; same offsets)
__device__ __forceinline__ void tile_carve(Tile &tile, unsigned char *ptr) {
  const int npc = tile.npc;
  tile.I = (double *)ptr;
  ptr += sizeof(double) * tile.R * npc;
  tile.L = (double *)ptr;
  ptr += sizeof(double) * tile.R * npc;
  tile.Agpu = (double *)ptr;
  ptr += sizeof(double) * npc;
  tile.Acpu = (double *)ptr;
  ptr += sizeof(double) * npc;
  tile.gpu_count = (double *)ptr;
  ptr += sizeof(double) * npc;
  tile.rank = (int *)ptr;
  ptr += sizeof(int) * npc;
  tile.flags = (uint32_t *)ptr;
  ptr += sizeof(uint32_t) * npc;
  tile.node = (int *)ptr;
  ptr += sizeof(int) * npc;
  tile.dom = (int *)ptr;
}

struct ScanShared {
  unsigned long long dw[kDecWords];
  Decision dec;
  Track trk[2];
  int kind, n_delta, batching, xbits;
  int pref_level;                           // topology node scoring: global level index or -1 (off)
  unsigned char dom_bucket[kDomBuckets];    // bucket per preferred-level domain, 255 = no entry
  int2 delta[kMaxDelta];
  unsigned int mine_bits[kMaxDelta / 32], ext_bits[kMaxDelta / 32];  // per 32 list entries: owned by this scanner / extended
  int fit_count;
  int ext_dirty;  // the preferred-level score table changed in this launch
  int excl[kTopM];
  Cand cands[kTopM];
  double dreq[kMaxDelta][KAI_MAX_RES];
  int dln[kMaxDelta];
};


// One launch = one decision record (`lrec`, kernel parameter).  The tile lives in global memory between launches, in
// the layout tile_carve() gives it; DK_LOAD fills it from the session tables, DK_DONE writes it back.  Returns true
// when the record asks for an answer (the caller then runs the last-CTA reduction).
__device__ bool scanner_main(const ActionParams &p, const LaunchRec *lrec, unsigned char *smem, Cand *sh_warp, double *sh_d,
                             int *sh_i, ScanShared &sh, Tile &tile) {
  const DevSnap &s = p.s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int my = (int)blockIdx.x;
  unsigned char *gstate = p.g_scan_state + (size_t)my * kScanStateBytes;
  const bool load_tile = (int)(lrec->dw[0] & 0xff) == DK_LOAD;
  if (tid == 0) {
    int npc = p.nodes_per_cta;
    unsigned char *ptr = p.g_tiles + (size_t)my * p.g_tile_stride;
    tile.npc = npc;
    tile.R = s.R;
    tile.nscan = p.scanners;
    tile.nscan_log2 = (tile.nscan > 0 && (tile.nscan & (tile.nscan - 1)) == 0) ? 31 - __clz(tile.nscan) : -1;
    tile.my = my;
    tile.nshard = p.cfg.shard_count;
    tile.shard = p.cfg.shard_rank;
    {
      long long first = (long long)my * tile.nshard + tile.shard, step = (long long)tile.nscan * tile.nshard;
      tile.count = first < s.N ? (int)((s.N - first + step - 1) / step) : 0;
    }
    tile.n_dom_levels = p.node_domain ? p.n_dom_levels : 0;
    tile_carve(tile, ptr);
    sh.pref_level = -1;
    sh.ext_dirty = 0;
    if (!load_tile) sh.pref_level = *(const int *)gstate;
  }
  __syncthreads();
  if (!load_tile && sh.pref_level >= 0)  // the score buckets of the preferred level persist between launches
    for (int i = tid; i < kDomBuckets; i += blockDim.x) sh.dom_bucket[i] = gstate[16 + i];
  if (load_tile) {
    for (int ln = tid; ln < tile.count; ln += blockDim.x) {
      const int rk = tile_row_rank(tile, ln);
      const int n = s.rank_to_node[rk];
      tile.node[ln] = n;
      for (int r = 0; r < s.R; r++) {
        tile.I[r * tile.npc + ln] = s.idle[(size_t)r * s.N + n];
        tile.L[r * tile.npc + ln] = s.rel[(size_t)r * s.N + n];
      }
      tile.Agpu[ln] = s.alloc[(size_t)KAI_RES_GPU * s.N + n];
      tile.Acpu[ln] = s.alloc[(size_t)KAI_RES_CPU * s.N + n];
      tile.gpu_count[ln] = s.gpu_count[n];
      tile.rank[ln] = rk;
      tile.flags[ln] = s.nflags[n];
      for (int l = 0; l < tile.n_dom_levels; l++) tile.dom[l * tile.npc + ln] = p.node_domain[(size_t)l * s.N + n];
    }
    __syncthreads();
    if (tid == 0) *(int *)gstate = -1;
    return false;
  }
  const unsigned long long seq = lrec->seq;
  long long ts[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  long long c0 = clock64();
  if (tid < kDecWords) sh.dw[tid] = lrec->dw[tid];
  __syncthreads();
  long long c1 = clock64();
  if (tid < 32) {  // decode in parallel: lane r writes req[r], lanes 8/9 the trackers, lane 10 the scalars
    const unsigned long long w0 = sh.dw[0];
    const unsigned int bits = (unsigned int)((w0 >> 24) & 0xff);
    Decision &d = sh.dec;
    if (tid < KAI_MAX_RES) d.req[tid] = __longlong_as_double((long long)sh.dw[2 + tid]);
    if (tid == 8 || tid == 9) {
      const int k = tid - 8;
      sh.trk[k].mn = __longlong_as_double((long long)sh.dw[10 + 2 * k]);
      sh.trk[k].mx = __longlong_as_double((long long)sh.dw[11 + 2 * k]);
      sh.trk[k].cnt_mn = (int)(unsigned int)(sh.dw[14 + k] & 0xffffffffu);
      sh.trk[k].cnt_mx = (int)(unsigned int)(sh.dw[14 + k] >> 32);
      sh.trk[k].dirty = (bits & (k == 0 ? DB_DIRTY0 : DB_DIRTY1)) ? 1 : 0;
    }
    if (tid == 10) {
      sh.kind = (int)(w0 & 0xff);
      d.res = (int)((w0 >> 8) & 0xff);
      d.strategy = (int)((w0 >> 16) & 0xff);
      sh.n_delta = (int)((w0 >> 32) & 0xffff);
      sh.xbits = (int)((w0 >> 48) & 0xffff);
      d.restricted = (sh.xbits & XB_RESTRICT) ? 1 : 0;
      d.gpu_task = (bits & DB_GPU_TASK) ? 1 : 0;
      d.best_effort = (bits & DB_BEST_EFFORT) ? 1 : 0;
      d.pipeline_only = (bits & DB_PIPELINE_ONLY) ? 1 : 0;
      sh.batching = (bits & DB_BATCHING) ? 1 : 0;
      d.nominated = (int)(unsigned int)(sh.dw[1] & 0xffffffffu);
      d.pred_class = (int)(unsigned int)(sh.dw[1] >> 32);
      const int tk = d.res == KAI_RES_GPU ? 0 : 1;
      d.mn = __longlong_as_double((long long)sh.dw[10 + 2 * tk]);
      d.mx = __longlong_as_double((long long)sh.dw[11 + 2 * tk]);
      d.task = -1;
    }
  }
  __syncthreads();
  long long c2 = clock64();
  // ---- apply the node deltas that belong to this tile (loads in parallel, application in list order) ----
  // Every scanner sees the whole list but owns ~1/scanners of it: the entries are classified in parallel (ballot bits
  // per 32 entries: "mine", "extended") and only the set bits are walked, in list order.
  const int nd = sh.n_delta;
  if (nd > 0) {
    for (int e0 = 0; e0 < nd; e0 += blockDim.x) {
      const int e = e0 + tid;
      bool mine = false, ext = false;
      if (e < nd) {
        const unsigned long long lo = (unsigned long long)lrec->dkey[e] | ((unsigned long long)lrec->dtask[e] << 32);
        int2 en = make_int2((int)(unsigned int)(lo & 0xffffffffu), (int)(unsigned int)(lo >> 32));
        sh.delta[e] = en;
        int ln = 0;
        ext = en.x < 0;
        mine = en.x >= 0 && tile_owns(tile, (unsigned int)(en.x & 0x0fffffff), ln) && ln < tile.count;
        sh.dln[e] = ln | ((int)lrec->dcount[e] << 24);  // repeat count - 1 in the top byte
        if (mine && ((en.x >> 28) & 7) < ND_FEAS_SET)
          for (int r = 0; r < s.R; r++) sh.dreq[e][r] = __ldg(&s.t_req[(size_t)en.y * s.R + r]);
      }
      const unsigned int mb = __ballot_sync(0xffffffffu, mine), xb = __ballot_sync(0xffffffffu, ext);
      if (lane == 0) {
        sh.mine_bits[(e0 >> 5) + warp] = mb;
        sh.ext_bits[(e0 >> 5) + warp] = xb;
      }
    }
    __syncthreads();
    const int n_words = (nd + 31) >> 5;
    if (warp == 0 && lane < s.R) {
      for (int w = 0; w < n_words; w++) {
        unsigned int bits = sh.mine_bits[w];
        while (bits) {
          const int e = (w << 5) + __ffs((int)bits) - 1;
          bits &= bits - 1;
          int2 en = sh.delta[e];
          const int ln = sh.dln[e] & 0xffffff, reps = ((unsigned int)sh.dln[e] >> 24) + 1;
          const int code = (en.x >> 28) & 7;
          if (code >= ND_FEAS_SET) {
            if (lane == 0) tile.flags[ln] = code == ND_FEAS_SET ? (tile.flags[ln] | kTileFeas) : (tile.flags[ln] & ~kTileFeas);
            continue;
          }
          for (int k = 0; k < reps; k++)
            apply_delta_row(tile.I[lane * tile.npc + ln], tile.L[lane * tile.npc + ln], code, sh.dreq[e][lane]);
        }
      }
    }
    __syncthreads();
    // extended entries, in list order: topology domain selection (each thread its own rows) and the per-domain
    // score table (thread 0; the clearing BEGIN is the only step the others take part in)
    bool any_ext = false;
    for (int w = 0; w < n_words; w++) {
      unsigned int bits = sh.ext_bits[w];
      while (bits) {
        const int e = (w << 5) + __ffs((int)bits) - 1;
        bits &= bits - 1;
        any_ext = true;
        const int2 en = sh.delta[e];
        const int kind = (en.x >> 28) & 7;
        const unsigned int a = (unsigned int)en.x & 0x0fffffffu, b = (unsigned int)en.y;
        if (kind == EXT_SELECT || kind == EXT_SELECT_ROOT) {
          const int slot = kind == EXT_SELECT ? (int)((a >> 8) & 7u) : (int)((a >> 16) & 7u);
          const uint32_t bit = kTileDom >> slot;
          for (int ln = tid; ln < tile.count; ln += blockDim.x) {
            bool in;
            if (kind == EXT_SELECT) {
              in = tile.dom[((int)(a & 0xffu) - 1) * tile.npc + ln] == (int)b;
            } else {
              in = true;
              for (int l = (int)(a & 0xff); l < (int)((a >> 8) & 0xff); l++)
                if (tile.dom[l * tile.npc + ln] < 0) in = false;
            }
            tile.flags[ln] = in ? (tile.flags[ln] | bit) : (tile.flags[ln] & ~bit);
          }
        } else if (kind == EXT_SCORE_BEGIN) {
          __syncthreads();  // earlier EXT_SCORE writes of thread 0 precede the clearing
          for (int i = tid; i < kDomBuckets; i += blockDim.x) sh.dom_bucket[i] = 255;
          if (tid == 0) sh.pref_level = (int)a, sh.ext_dirty = 1;
          __syncthreads();
        } else if (kind == EXT_SCORE) {
          if (tid == 0 && a < (unsigned int)kDomBuckets) sh.dom_bucket[a] = (unsigned char)b, sh.ext_dirty = 1;
        } else if (kind == EXT_SCORE_END) {
          if (tid == 0) sh.pref_level = -1, sh.ext_dirty = 1;
        }
      }
    }
    if (any_ext) __syncthreads();
  }
  if (sh.xbits & (XB_SNAP_ALL | XB_SNAP_GPUFREE)) {  // common.FeasibleNodesForJob (feasible_nodes.go:11-26)
    const bool all = (sh.xbits & XB_SNAP_ALL) != 0;
    for (int ln = tid; ln < tile.count; ln += blockDim.x) {
      bool in = all || tile.I[KAI_RES_GPU * tile.npc + ln] > 0 || tile.L[KAI_RES_GPU * tile.npc + ln] > 0;
      tile.flags[ln] = in ? (tile.flags[ln] | kTileFeas) : (tile.flags[ln] & ~kTileFeas);
    }
    __syncthreads();
  }
  long long c3 = clock64();
  const int kind = sh.kind;
  const bool done = kind == DK_DONE || ((volatile long long *)p.counters)[24] != 0;
  if (!done) {
    if (kind == DK_SCAN || kind == DK_TOPK || kind == DK_MINMAX) {
      // the sweep reads every row several times (top-M passes, repeat analysis): stage this scanner's block of g_tiles
      // in shared memory with one pass of independent 16-byte loads; deltas and row flags were applied to the
      // global copy above, nothing below writes the tile
      const uint4 *src = (const uint4 *)(p.g_tiles + (size_t)my * p.g_tile_stride);
      uint4 *dst = (uint4 *)smem;
      const int n16 = (int)(p.tile_bytes >> 4);
      for (int i = tid; i < n16; i += blockDim.x) dst[i] = src[i];
      if (tid == 0) tile_carve(tile, smem);
      __syncthreads();
    }
    unsigned long long *slot = p.xbuf + (size_t)my * kSlotWords;
    if (!p.fused_in_kernel && kind == DK_SCAN && (sh.xbits & XB_FUSED_MM)) {
      // the extremes of this row set were reduced by the MINMAX launch that precedes this one on the stream
      if (tid == 0) {
        const int k = sh.dec.res == KAI_RES_GPU ? 0 : 1;
        sh.dec.mn = p.mm_result[2 * k];
        sh.dec.mx = p.mm_result[2 * k + 1];
      }
      __syncthreads();
    } else if (kind == DK_SCAN && (sh.xbits & XB_FUSED_MM)) {
      {
        // pack.go:66-86 over the current node set: local extremes -> device slots -> every scanner reduces all slots
        double mn[2], mx[2];
        tile_extremes(tile, sh.dec.restricted, sh.xbits, sh_d, mn, mx);
        // the one wait inside a launch: every scanner's extremes, tagged with the full sequence number (a slot of an
        // earlier record never matches), under the watchdog so that a protocol bug ends the kernel
        unsigned long long *mmbase = p.mmbuf;
        if (tid < 4) {
          const double v = tid == 0 ? mn[0] : tid == 1 ? mx[0] : tid == 2 ? mn[1] : mx[1];
          st_relaxed_b128(mmbase + (size_t)my * kSlotWords + 2 * tid, (unsigned long long)__double_as_longlong(v),
                          seq);
        }
        __syncthreads();
        double g[4] = {DBL_MAX, 0.0, DBL_MAX, 0.0};
        for (int c = tid; c < p.scanners; c += blockDim.x)
          for (int i = 0; i < 4; i++) {
            unsigned long long lo, hi;
            Spin spin;
            do {
              ld_relaxed_b128(mmbase + (size_t)c * kSlotWords + 2 * i, lo, hi);
            } while (hi != seq && !spin.expired(p, 14, seq, c));
            double v = __longlong_as_double((long long)lo);
            g[i] = i & 1 ? fmax(g[i], v) : fmin(g[i], v);
          }
        for (int i = 0; i < 4; i++)
          for (int o = 16; o > 0; o >>= 1) {
            double ov = __shfl_xor_sync(0xffffffffu, g[i], o);
            g[i] = i & 1 ? fmax(g[i], ov) : fmin(g[i], ov);
          }
        if (lane == 0)
          for (int i = 0; i < 4; i++) sh_d[16 + warp * 4 + i] = g[i];
        __syncthreads();
        if (tid == 0) {
          for (int w = 1; w < nw; w++)
            for (int i = 0; i < 4; i++)
              g[i] = i & 1 ? fmax(g[i], sh_d[16 + w * 4 + i]) : fmin(g[i], sh_d[16 + w * 4 + i]);
          const int k = sh.dec.res == KAI_RES_GPU ? 0 : 1;
          sh.dec.mn = g[2 * k];
          sh.dec.mx = g[2 * k + 1];
        }
        __syncthreads();
      }
    }
    // the placement sweep's key of a row: row set, predicate mask, FittingNode + NodeOrderFn, topology term
    const Decision &dec = sh.dec;
    const uint32_t *mask = dec.pred_class >= 0 ? s.pred_mask + (size_t)dec.pred_class * s.mask_words : nullptr;
    const int xbits = sh.xbits, pref_level = sh.pref_level;
    auto place_key = [&](int ln, double &score) {
      const int n = tile.node[ln];
      if (!in_row_set(tile, ln, dec.restricted, xbits)) return false;
      if (mask && !((__ldg(&mask[n >> 5]) >> (n & 31)) & 1u)) return false;
      bool fit_i;
      if (!node_key(dec, tile.R, tile.I + ln, tile.L + ln, tile.npc, tile.Agpu[ln], tile.Acpu[ln], tile.gpu_count[ln],
                    tile.flags[ln], n, score, fit_i))
        return false;
      if (pref_level >= 0) {  // topology/node_scoring.go:17-53, the last NodeOrderFn of the default tiers
        const int dd = tile.dom[pref_level * tile.npc + ln];
        const unsigned char bk = (dd >= 0 && dd < kDomBuckets) ? sh.dom_bucket[dd] : (unsigned char)255;
        if (bk == 255) return false;  // no entry: NodeOrderFn fails, the node is dropped (session.go:247-251)
        score = __dadd_rn(score, __dmul_rn((double)bk, 10000.0));
      }
      return true;
    };
    if (kind == DK_SCAN && p.topm && !(sh.xbits & XB_SINGLE)) {
      // ---- top-M answer into device lines (k_merge_cluster merges them; no last-CTA reduction) ----
      scan_top_m(tile, place_key, sh_warp, sh.excl, sh.cands, &sh.fit_count);
      if (tid == 0) ts[4] += clock64() - c3;
      unsigned long long *lines = p.d_list + (size_t)my * kListLines * kListLineWords;
      if (warp < kTopM) {
        double topo_term = 0.0;
        if (sh.pref_level >= 0 && sh.cands[warp].rank != kRankNone) {
          const int dd = tile.dom[sh.pref_level * tile.npc + sh.cands[warp].ln];
          topo_term = __dmul_rn((double)((dd >= 0 && dd < kDomBuckets) ? sh.dom_bucket[dd] : 0), 10000.0);
        }
        publish_list_candidate(tile, sh.dec, sh.cands[warp], sh.fit_count > kTopM, lines + 2 * warp,
                               lines + (size_t)(1 + warp) * kListLineWords, topo_term);
      }
    } else if (kind == DK_TOPK) {
      // ---- accumulated_scenario_filters/idle_gpus: rows by idle + releasing GPUs, descending (name rank ascending
      //      among equals), strictly after the cutoff (req[0] = key, req[1] = rank, req[2] = cutoff present) ----
      const bool has_cut = dec.req[2] != 0.0;
      const double cut_key = dec.req[0];
      const uint32_t cut_rank = (uint32_t)dec.req[1];
      auto idle_gpu_key = [&](int ln, double &key) {
        key = __dadd_rn(tile.I[KAI_RES_GPU * tile.npc + ln], tile.L[KAI_RES_GPU * tile.npc + ln]);
        const uint32_t rk = (uint32_t)tile.rank[ln];
        return !has_cut || key < cut_key || (key == cut_key && rk > cut_rank);
      };
      scan_top_m(tile, idle_gpu_key, sh_warp, sh.excl, sh.cands, &sh.fit_count);
      unsigned long long *lines = p.d_list + (size_t)my * kListLines * kListLineWords;
      if (tid < kTopM) {
        const Cand c = sh.cands[tid];
        const uint32_t flags = sh.fit_count > kTopM ? LF_MORE : 0u;
        unsigned long long hi = ((unsigned long long)flags << 32) | (unsigned long long)(c.rank == kRankNone ? kRankNone : (c.rank & 0xffffffu));
        st_relaxed_sys_b128(lines + 2 * tid, (unsigned long long)__double_as_longlong(c.score), hi);
      }
    } else if (kind == DK_SCAN) {
      Cand local = scan_tile(tile, place_key, sh_warp, nullptr, 0, nullptr);
      long long c4 = clock64();
      if (tid == 0) ts[4] += c4 - c3;
      if (warp == 0) publish_candidate(sh.trk, tile, sh.dec, local, slot, sh.batching);
    } else if (kind == DK_MINMAX) {
      double mn[2], mx[2];
      tile_extremes(tile, dec.restricted, xbits, sh_d, mn, mx);
      int c[4] = {0, 0, 0, 0};
      for (int ln = tid; ln < tile.count; ln += blockDim.x)
        for (int k = 0; k < 2; k++) {
          int res = k == 0 ? KAI_RES_GPU : KAI_RES_CPU;
          double overall = k == 0 ? tile.Agpu[ln] : tile.Acpu[ln];
          if (overall == 0) continue;
          if (!in_row_set(tile, ln, dec.restricted, xbits)) continue;
          double cur = __dadd_rn(tile.I[res * tile.npc + ln], tile.L[res * tile.npc + ln]);
          if (cur == mn[k]) c[2 * k]++;
          if (cur == mx[k]) c[2 * k + 1]++;
        }
      for (int i = 0; i < 4; i++)
        for (int o = 16; o > 0; o >>= 1) c[i] += __shfl_xor_sync(0xffffffffu, c[i], o);
      if (lane == 0)
        for (int i = 0; i < 4; i++) sh_i[warp * 4 + i] = c[i];
      __syncthreads();
      if (tid == 0) {
        int tot[4] = {0, 0, 0, 0};
        for (int w = 0; w < nw; w++)
          for (int i = 0; i < 4; i++) tot[i] += sh_i[w * 4 + i];
        st_relaxed_b128(slot + 0, (unsigned long long)__double_as_longlong(mn[0]), (unsigned long long)(unsigned int)tot[0]);
        st_relaxed_b128(slot + 2, (unsigned long long)__double_as_longlong(mx[0]), (unsigned long long)(unsigned int)tot[1]);
        st_relaxed_b128(slot + 4, (unsigned long long)__double_as_longlong(mn[1]), (unsigned long long)(unsigned int)tot[2]);
        st_relaxed_b128(slot + 6, (unsigned long long)__double_as_longlong(mx[1]), (unsigned long long)(unsigned int)tot[3]);
      }
    }
    if (tid == 0) {
      long long c5 = clock64();
      ts[1] += c1 - c0;  // poll + words
      ts[2] += c2 - c1;  // decode
      ts[3] += c3 - c2;  // deltas
      ts[5] += c5 - c3;  // scan + publish
      ts[6]++;
    }
    __syncthreads();
  }
  if (tid == 0 && my == 0)  // launches of one action follow each other on the stream: plain accumulation
    for (int i = 0; i < 7; i++) p.counters[32 + i] += ts[i];
  if (sh.ext_dirty) {  // preferred-level score table of this scanner: back to its global copy
    for (int i = tid; i < kDomBuckets; i += blockDim.x) gstate[16 + i] = sh.dom_bucket[i];
    if (tid == 0) *(int *)gstate = sh.pref_level;
  }
  if (!done) return kind != DK_FLUSH;
  // ---- DONE: write the tile back to the session tables ----
  for (int ln = tid; ln < tile.count; ln += blockDim.x) {
    int n = tile.node[ln];
    for (int r = 0; r < s.R; r++) {
      s.idle[(size_t)r * s.N + n] = tile.I[r * tile.npc + ln];
      s.rel[(size_t)r * s.N + n] = tile.L[r * tile.npc + ln];
    }
  }
  return false;
}

// =============================================================================================
// the last CTA of a launch
// =============================================================================================
// Reduce the scanners' answers for record `seq` on the GPU and write ONE 64-byte line to host memory (a host
// core pays ~80 ns per GPU-written cache line it reads; 147 lines per sweep were the bottleneck).  The scanners wrote
// their slots before taking the ticket, so they are read once.  The line is the payload, then, after a system fence,
// the sequence number in its last word.
__device__ void reduce_answers(const ActionParams &p, int kind, unsigned long long seq) {
  const int lane = threadIdx.x & 31;
  const int n = p.scanners;
  const unsigned long long *buf = p.xbuf;
  unsigned long long *out = (kind == DK_SCAN ? p.h_slot : p.h_mmslot) + (size_t)(seq & 1) * p.cfg.shard_count * kLineWords;
  if (kind == DK_SCAN) {
    Cand best = {-1.0, kRankNone, -1};  // ln: the winner's slot
    for (int c = lane; c < n; c += 32) {
      unsigned long long lo, hi;
      ld_relaxed_b128(buf + (size_t)c * kSlotWords, lo, hi);
      double sc = __longlong_as_double((long long)lo);
      uint32_t rk = (uint32_t)(hi & 0xffffffu);
      if (better(sc, rk, best.score, best.rank)) best = {sc, rk, c};
    }
    best = warp_argmax(best);
    if (lane == 0) {  // the winning slot's meta word, cur_a values and repeat events
      unsigned long long meta = (unsigned long long)kRankNone, ag = 0, ac = 0, rep = 0, unused;
      if (best.rank != kRankNone) {
        const unsigned long long *slot = buf + (size_t)best.ln * kSlotWords;
        ld_relaxed_b128(slot, unused, meta);
        ld_relaxed_b128(slot + 2, ag, ac);
        if ((meta >> 24) & 0xffu) ld_relaxed_b128(slot + 4, rep, unused);
      }
      st_relaxed_sys_b128(out, (unsigned long long)__double_as_longlong(best.score), meta);
      st_relaxed_sys_b128(out + 2, ag, ac);
      st_relaxed_sys_b128(out + 4, rep, 0ull);
    }
  } else if (kind == DK_MINMAX) {
    double gmn[2] = {DBL_MAX, DBL_MAX}, gmx[2] = {0, 0};
    long long cmn[2] = {0, 0}, cmx[2] = {0, 0};
    for (int cta = lane; cta < n; cta += 32) {
      const unsigned long long *slot = buf + (size_t)cta * kSlotWords;
      for (int k = 0; k < 2; k++) {
        unsigned long long lo, hi;
        ld_relaxed_b128(slot + 4 * k, lo, hi);
        merge_extreme(gmn[k], cmn[k], __longlong_as_double((long long)lo), (int)(hi & 0xffffffffu), true);
        ld_relaxed_b128(slot + 4 * k + 2, lo, hi);
        merge_extreme(gmx[k], cmx[k], __longlong_as_double((long long)lo), (int)(hi & 0xffffffffu), false);
      }
    }
    for (int k = 0; k < 2; k++)
      for (int o = 16; o > 0; o >>= 1) {
        double omn = __shfl_xor_sync(0xffffffffu, gmn[k], o);
        long long ocmn = __shfl_xor_sync(0xffffffffu, cmn[k], o);
        double omx = __shfl_xor_sync(0xffffffffu, gmx[k], o);
        long long ocmx = __shfl_xor_sync(0xffffffffu, cmx[k], o);
        merge_extreme(gmn[k], cmn[k], omn, ocmn, true);
        merge_extreme(gmx[k], cmx[k], omx, ocmx, false);
      }
    if (lane == 0) {
      unsigned long long cnt[2];
      for (int k = 0; k < 2; k++) {
        p.mm_result[2 * k] = cmn[k] > 0 ? gmn[k] : DBL_MAX;  // the next launch (XB_FUSED_MM sweep) reads the extremes
        p.mm_result[2 * k + 1] = cmx[k] > 0 ? gmx[k] : 0.0;
        const unsigned int c0 = (unsigned int)(cmn[k] > 0x7fffffff ? 0x7fffffff : cmn[k]);
        const unsigned int c1 = (unsigned int)(cmx[k] > 0x7fffffff ? 0x7fffffff : cmx[k]);
        cnt[k] = (unsigned long long)c0 | ((unsigned long long)c1 << 32);
      }
      // {gpu min, gpu max} {cpu min, cpu max} {gpu counts at min | at max << 32, cpu counts}
      st_relaxed_sys_b128(out, (unsigned long long)__double_as_longlong(gmn[0]), (unsigned long long)__double_as_longlong(gmx[0]));
      st_relaxed_sys_b128(out + 2, (unsigned long long)__double_as_longlong(gmn[1]), (unsigned long long)__double_as_longlong(gmx[1]));
      st_relaxed_sys_b128(out + 4, cnt[0], cnt[1]);
    }
  }
  if (lane == 0) {
    __threadfence_system();  // the payload is out before the sequence number
    st_relaxed_sys_b128(out + kLineWords - 2, 0ull, seq);
  }
  __syncwarp();
}

// =============================================================================================
// list answers: merge of the scanners' top-M candidates
// =============================================================================================
// Integer sort keys of a candidate: h = list_key(score) (ascending h is descending score for any non-NaN score: DK_TOPK
// scores, Idle + Releasing GPUs, go negative on over-committed nodes; -0.0 and +0.0 share a key), l = rank << 32 |
// source (scanner * kTopM + m); an empty slot is all ones in both and sorts last.
constexpr int kMergeThreads = 1024;  // one candidate per thread: scanners x kTopM <= 1024
__device__ __forceinline__ bool mk_before(unsigned long long ah, unsigned long long al, unsigned long long bh, unsigned long long bl) {
  return ah < bh || (ah == bh && al < bl);
}
// Merge kernel, launched right after a list sweep on the same stream: sorts the scanners' top-M candidates (device lines
// of d_list) by (score desc, name rank asc) with a bitonic network, cuts the list where an unseen row could be better
// (the best "last reported key" among scanners that have more fitting rows than they reported) and streams the usable
// prefix as 48-byte entries {score, meta, Ig, Lg, Ic, Lc} + one header word to host memory: the host reads one
// contiguous list instead of scanners x (1 + M) cache lines.
//
// It runs on a thread-block cluster (Hopper: 4 CTAs x 256 threads on 4 SMs, one candidate per thread): the
// 55-step network is bound by instruction issue, so four SMs share it instead of one.  Partner exchange: warp shuffle
// below 32 lanes, the CTA's shared memory below 256, the partner CTA's shared memory (distributed shared memory,
// cluster.map_shared_rank) for the three steps with j >= 256; every CTA streams its own quarter of the sorted prefix to
// host memory, CTA 0 writes the header after the cluster barrier.
constexpr int kMergeCtas = 4, kMergeCtaThreads = kMergeThreads / kMergeCtas;
constexpr size_t kMergeCtaSmemBytes = (size_t)kMergeCtaThreads * 8 * (2 + kCEntryWords);
__global__ void __cluster_dims__(kMergeCtas, 1, 1) __launch_bounds__(kMergeCtaThreads, 1)
    k_merge_cluster(const __grid_constant__ ActionParams p, unsigned long long seq, int with_payload) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char dyn_smem[];
  unsigned long long *xh = (unsigned long long *)dyn_smem, *xl = xh + kMergeCtaThreads, *stage = xl + kMergeCtaThreads;
  __shared__ unsigned long long cut_h[kMergeCtaThreads / 32];
  __shared__ unsigned int cut_r[kMergeCtaThreads / 32];
  __shared__ int n_ok[kMergeCtaThreads / 32];
  __shared__ unsigned long long cta_cut_h;  // read by the other CTAs of the cluster
  __shared__ unsigned int cta_cut_r;
  __shared__ int cta_n_ok;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned int crank = cluster.block_rank();
  const int g = (int)crank * kMergeCtaThreads + tid;  // my position in the network
  const int n_scan = p.scanners;
  const int n_c = n_scan * kTopM;
  const unsigned long long *base = p.d_list;
  const long long t0 = clock64();
  unsigned long long h = ~0ull, l = ~0ull;
  bool more = false;
  if (g < n_c) {
    const int c = g / kTopM, m = g % kTopM;
    const unsigned long long *lines = base + (size_t)c * kListLines * kListLineWords;
    const uint4 v = __ldcg((const uint4 *)(lines + 2 * m));
    const unsigned long long lo = (unsigned long long)v.x | ((unsigned long long)v.y << 32);
    const unsigned long long hi = (unsigned long long)v.z | ((unsigned long long)v.w << 32);
    const uint32_t rank = (uint32_t)(hi & 0xffffffu);
    more = (((uint32_t)(hi >> 32) & 0xffu) & LF_MORE) != 0;
    if (rank != kRankNone) {
      h = list_key(__longlong_as_double((long long)lo));
      l = ((unsigned long long)rank << 32) | (unsigned long long)g;
    }
  }
  static_assert(kTopM == 4, "the group reductions below assume 4 candidates per scanner");
  const unsigned int grp = 0xfu << (lane & ~3);
  const bool any_more = (__ballot_sync(0xffffffffu, more) & grp) != 0;
  const unsigned int real = __ballot_sync(0xffffffffu, l != ~0ull) & grp;
  unsigned long long ch = ~0ull;
  unsigned int cr = kRankNone;
  if (any_more && real && lane == 31 - __clz((int)real)) {
    ch = h;
    cr = (unsigned int)(l >> 32);
  }
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long oh = __shfl_xor_sync(0xffffffffu, ch, o);
    const unsigned int orr = __shfl_xor_sync(0xffffffffu, cr, o);
    if (orr != kRankNone && (cr == kRankNone || oh < ch || (oh == ch && orr < cr))) {
      ch = oh;
      cr = orr;
    }
  }
  if (lane == 0) {
    cut_h[warp] = ch;
    cut_r[warp] = cr;
  }
  __syncthreads();
  if (tid == 0) {
    unsigned long long bh = ~0ull;
    unsigned int br = kRankNone;
    for (int w = 0; w < kMergeCtaThreads / 32; w++)
      if (cut_r[w] != kRankNone && (br == kRankNone || cut_h[w] < bh || (cut_h[w] == bh && cut_r[w] < br))) {
        bh = cut_h[w];
        br = cut_r[w];
      }
    cta_cut_h = bh;
    cta_cut_r = br;
  }
  const long long t1 = clock64();
  // ---- bitonic sort over the cluster, one element per thread ----
  for (int k = 2; k <= kMergeThreads; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      unsigned long long oh, ol;
      if (j < 32) {
        oh = __shfl_xor_sync(0xffffffffu, h, j);
        ol = __shfl_xor_sync(0xffffffffu, l, j);
      } else if (j < kMergeCtaThreads) {
        xh[tid] = h;
        xl[tid] = l;
        __syncthreads();
        oh = xh[tid ^ j];
        ol = xl[tid ^ j];
        __syncthreads();
      } else {  // the partner sits at the same thread index of CTA crank ^ (j / 256)
        xh[tid] = h;
        xl[tid] = l;
        cluster.sync();
        const unsigned int peer = crank ^ (unsigned int)(j / kMergeCtaThreads);
        const unsigned long long *rh = cluster.map_shared_rank(xh, peer), *rl = cluster.map_shared_rank(xl, peer);
        oh = rh[tid];
        ol = rl[tid];
        cluster.sync();
      }
      const bool lower = (g & j) == 0;
      const bool up = (g & k) == 0;
      const bool take = (lower == up) ? mk_before(oh, ol, h, l) : mk_before(h, l, oh, ol);
      if (take) {
        h = oh;
        l = ol;
      }
    }
  cluster.sync();  // every CTA's cut candidate is written; the exchange planes are free
  const long long t2 = clock64();
  unsigned long long gh = ~0ull;
  unsigned int gr = kRankNone;
  for (unsigned int c = 0; c < (unsigned int)kMergeCtas; c++) {
    const unsigned long long oh = *cluster.map_shared_rank(&cta_cut_h, c);
    const unsigned int orr = *cluster.map_shared_rank(&cta_cut_r, c);
    if (orr != kRankNone && (gr == kRankNone || oh < gh || (oh == gh && orr < gr))) {
      gh = oh;
      gr = orr;
    }
  }
  const bool have_cut = gr != kRankNone;
  const unsigned int my_rank = (unsigned int)(l >> 32);
  const bool ok = l != ~0ull && (!have_cut || h < gh || (h == gh && my_rank <= gr));
  const unsigned int okb = __ballot_sync(0xffffffffu, ok);
  if (lane == 0) n_ok[warp] = __popc(okb);
  __syncthreads();
  if (tid == 0) {
    int t = 0;
    for (int w = 0; w < kMergeCtaThreads / 32; w++) t += n_ok[w];
    cta_n_ok = t;
  }
  cluster.sync();
  int n_out = 0;
  for (unsigned int c = 0; c < (unsigned int)kMergeCtas; c++) n_out += *cluster.map_shared_rank(&cta_n_ok, c);
  unsigned long long *out = p.h_clist + (size_t)(seq & 1) * kCListWords;
  // this CTA's quarter of the sorted list: positions [crank * 256, crank * 256 + 256) below n_out
  if (g < n_out) {
    const int src = (int)(l & 0xffffffffu);
    const int c = src / kTopM, m = src % kTopM;
    const unsigned long long *lines = base + (size_t)c * kListLines * kListLineWords;
    const uint4 v = __ldcg((const uint4 *)(lines + 2 * m));
    unsigned long long *e = stage + (size_t)tid * kCEntryWords;
    e[0] = (unsigned long long)v.x | ((unsigned long long)v.y << 32);
    e[1] = (unsigned long long)v.z | ((unsigned long long)v.w << 32);
    for (int q = 2; q < kCEntryWords; q++) e[q] = 0;
    if (with_payload) {  // {Ig, Lg} {Ic, Lc}
      const ulonglong2 *pl = (const ulonglong2 *)(lines + (size_t)(1 + m) * kListLineWords);
      const ulonglong2 g = __ldcg(pl), c2 = __ldcg(pl + 1);
      e[2] = g.x;
      e[3] = g.y;
      e[4] = c2.x;
      e[5] = c2.y;
    }
  }
  __syncthreads();
  const int first = (int)crank * kMergeCtaThreads;
  const int mine = max(0, min(n_out - first, kMergeCtaThreads));
  const int n16 = (mine * kCEntryWords) / 2;
  unsigned long long *out_mine = out + 2 + (size_t)first * kCEntryWords;
  for (int i = tid; i < n16; i += kMergeCtaThreads) st_relaxed_sys_b128(out_mine + 2 * (size_t)i, stage[2 * i], stage[2 * i + 1]);
  __threadfence_system();  // my entries are out before the cluster barrier lets CTA 0 write the header
  cluster.sync();
  if (crank == 0 && tid == 0) {
    __threadfence_system();
    st_relaxed_sys_b128(out, (unsigned long long)(unsigned int)n_out | (have_cut ? (1ull << 31) : 0ull), seq);
    const long long t3 = clock64();
    p.counters[44] += t3 - t0;
    p.counters[45] += 1;
    p.counters[46] += t2 - t1;  // sort
    p.counters[39] += t1 - t0;  // candidate loads + cut
    p.counters[31] += t3 - t2;  // prefix, payload, stream out, header
  }
}

// Asks for 5 resident CTAs per SM, which caps the budget at 102 registers.  Left to its default, ptxas settles on 80
// registers and spills about 300 B per thread to local memory; with the bound it uses 96 registers and no spills.
__global__ void __launch_bounds__(kThreads, 5) k_record(const __grid_constant__ ActionParams p, const __grid_constant__ LaunchRec rec) {
  extern __shared__ __align__(16) unsigned char smem[];  // merge keys of the last CTA
  __shared__ Tile tile;
  __shared__ ScanShared scan_sh;
  __shared__ Cand sh_warp[kThreads / 32];
  __shared__ double sh_d[(kThreads / 32) * 8];
  __shared__ int sh_i[(kThreads / 32) * 4];
  __shared__ int is_last;
  const bool answers = scanner_main(p, &rec, smem, sh_warp, sh_d, sh_i, scan_sh, tile);
  if (!answers) return;
  // list answers (top-M lines in device memory) are merged by k_merge_cluster, the next launch on the stream
  if (scan_sh.kind == DK_TOPK || (scan_sh.kind == DK_SCAN && p.topm && !(scan_sh.xbits & XB_SINGLE))) return;
  // ---- the last CTA to finish reduces the answers of all scanners and writes the result to host memory ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1 ? 1 : 0;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x == 0) *p.ticket = 0;  // the next launch follows in stream order
  const int kind = scan_sh.kind;
  if (threadIdx.x < 32) reduce_answers(p, kind, rec.seq);
}

}  // namespace kai