// kai_solver.cuh — reclaim and consolidation (victim selection) on the host-sequenced engine.
//
// Replaces: actions/reclaim/reclaim.go:46-143, actions/consolidation/consolidation.go:32-157 and the solver
// they share — actions/common/solvers/{job_solver,pod_scenario_builder,by_pod_solver}.go, scenario/*.go,
// accumulated_scenario_filters/idle_gpus/*.go, actions/common/{action,feasible_nodes,minimal_job_comparison}.go,
// plugins/proportion/reclaimable/** and proportion.go:131-240.
//
// Division of work (same as allocate): everything that is O(nodes) runs on the GPU —
//   * every allocateTask of every simulation is one restricted, pipeline-only sweep of the scanners' tiles
//     (DK_SCAN with XB_RESTRICT: fit on Idle+Releasing, NodeOrderFn score, argmax on (score, name rank)),
//     preceded by the binpack min/max exchange over the same node set (DK_MINMAX) — or, when that set is small, the
//     same computation on the host mirror (host_sweep);
//   * the feasible-node set of a job (FeasibleNodesForJob) is a per-row bit the scanners compute from their tiles
//     (XB_SNAP_*), later edited by ND_FEAS_SET/CLR deltas when victims' nodes join the set;
//   * the idle-GPU scenario filter's "k nodes with most idle+releasing GPUs" is a DK_TOPK sweep;
//   * evictions / pipelines / undo travel as node deltas to the scanner that owns the row —
// while the control flow (scenario accumulation, statements with undo chains, queue-share validators) runs on the
// host sequencer thread.  Go map iteration orders are resolved canonically (ascending node / job / queue index),
// like in the oracle.  Host-only code (never compiled for the device).
#pragma once
#include <array>
#include <algorithm>
#include <cmath>
#include <map>
#include <set>
#include <vector>

#include "kai_host_seq.cuh"

namespace kai {

// container/heap (Go) on a[0..n): the same sift sequence, so non-antisymmetric comparators pop in the same order.
// The storage belongs to the caller (JobsOrder keeps every heap of a tree in one arena); `less` is any callable.
struct HeapGo {
  template <class Less>
  static void up(int *a, int j, const Less &less) {
    for (;;) {
      int i = (j - 1) / 2;
      if (i == j || j <= 0 || !less(a[j], a[i])) break;
      std::swap(a[i], a[j]);
      j = i;
    }
  }
  template <class Less>
  static bool down(int *a, int i0, int n, const Less &less) {
    int i = i0;
    for (;;) {
      int j1 = 2 * i + 1;
      if (j1 >= n || j1 < 0) break;
      int j = j1, j2 = j1 + 1;
      if (j2 < n && less(a[j2], a[j1])) j = j2;
      if (!less(a[j], a[i])) break;
      std::swap(a[i], a[j]);
      i = j;
    }
    return i > i0;
  }
  template <class Less>
  static void push(int *a, int &n, int x, const Less &less) {  // a has room for n + 1 entries
    a[n] = x;
    up(a, n, less);
    n++;
  }
  template <class Less>
  static int pop(int *a, int &n, const Less &less) {
    const int m = n - 1;
    std::swap(a[0], a[m]);
    down(a, 0, m, less);
    n = m;
    return a[m];
  }
  template <class Less>
  static void fix(int *a, int n, int i, const Less &less) {
    if (!down(a, i, n, less)) up(a, i, less);
  }
};

struct SolverJobCache {  // tasks_to_allocate / its resource sum of one job or view
  bool tta_valid = false, res_valid = false;
  unsigned stamp = 0;  // session jobs: valid while equal to SolverScratch::job_epoch
  std::vector<int> tta;
  double res[QR] = {0, 0, 0};
};

// Per-node, per-job and per-task scratch of the solver kept by the engine across actions.  It is sized to the snapshot
// and invalidated by epoch stamps (an entry is live while its stamp equals the current epoch) rather than reassigned,
// so an action's set-up and each partial job pay for what they touch, not O(N + J + T).
struct SolverScratch {
  int N = -1, J = -1, T = -1;
  // attempt-start idle / releasing GPUs of the nodes touched since the attempt began
  std::vector<unsigned> node_stamp;
  std::vector<double> start_ig, start_lg;
  unsigned node_epoch = 0;
  std::vector<SolverJobCache> job_cache;  // live jobs (invalidated per action and on every status change)
  unsigned job_epoch = 0;
  // per task: the recorded victims of a partial job, the tasks an idle-GPU filter has accounted
  std::vector<unsigned> rec_stamp, seen_stamp;
  unsigned rec_epoch = 0, seen_epoch = 0;
  // slot 0 of a task's NodeInfo.PodInfos entries (node, status) for the tasks the action changed (slot_list); the
  // others' slot is still the snapshot's
  std::vector<int> n0, s0, slot_list;
  std::vector<unsigned> slot_stamp;
  unsigned slot_epoch = 0;

  void size_for(int n, int j, int t) {
    if (n != N) {
      node_stamp.assign(n, 0);
      start_ig.assign(n, 0);
      start_lg.assign(n, 0);
      node_epoch = 0;
      N = n;
    }
    if (j != J) {
      job_cache.assign(j, SolverJobCache());
      job_epoch = 0;
      J = j;
    }
    if (t != T) {
      rec_stamp.assign(t, 0);
      seen_stamp.assign(t, 0);
      n0.assign(t, -1);
      s0.assign(t, 0);
      slot_stamp.assign(t, 0);
      rec_epoch = seen_epoch = slot_epoch = 0;
      T = t;
    }
  }
  template <class S>
  static unsigned bump(unsigned &epoch, std::vector<S> &stamped, unsigned S::*field) {
    if (++epoch == 0) {  // wrapped: no stale stamp may match the new epoch
      for (S &x : stamped) x.*field = 0;
      epoch = 1;
    }
    return epoch;
  }
  static unsigned bump(unsigned &epoch, std::vector<unsigned> &stamps) {
    if (++epoch == 0) {
      std::fill(stamps.begin(), stamps.end(), 0u);
      epoch = 1;
    }
    return epoch;
  }
};

struct Solver {
  HostBackend &hb;
  Seq &seq;
  Ctl &ctl;
  const DevSnap &s;
  const kai_config &cfg;
  const int N, Q, J, S, T, R;
  bool use_signatures = false;
  const int *job_signature = nullptr;

  // ---- session state (engine-internal task numbering; tasks of a podset are stored in TaskOrderFn order) ----
  int *st, *tn;            // task status / node (host mirror arrays, written back by the engine)
  unsigned char *tvirt;    // PodInfo.IsVirtualStatus
  // NodeInfo.PodInfos keeps a clone per node: a task evicted from A and pipelined to B sits on both (slots 0 and 1); a
  // victim that an earlier action moved and this one evicts and re-places sits on three or more: `on_extra` holds the
  // (task, node, status) entries beyond the two slots (rare, linear look-up).  Slot 0 lives in the scratch (scr.n0 /
  // scr.s0) for the tasks this action changed; for the others it is the snapshot's (node if active-used, node status).
  SolverScratch &scr;
  std::vector<int> &on_node1, &on_status1;
  std::vector<std::array<int, 3>> &on_extra;
  double *qa, *qnp;        // queue allocated / allocated-non-preemptible [3][Q]
  // GPU column of the host mirror of Idle / Releasing (seq.mirror, node-major; point look-ups only)
  double Ig(int n) const { return seq.mirror[(size_t)n * 2 * R + KAI_RES_GPU]; }
  double Lg(int n) const { return seq.mirror[(size_t)n * 2 * R + R + KAI_RES_GPU]; }
  // attempt-start values of touched rows (FeasibleNodesForJob and the filter's base map read the state the
  // attempt started from): scr.start_ig / scr.start_lg, valid where scr.node_stamp equals scr.node_epoch

  enum { OPK_ALLOCATE = 0, OPK_PIPELINE = 1, OPK_EVICT = 2, OPK_UNDO = 3 };
  struct SOp {
    int kind, task, prev_status, prev_node, next_node, prev_virtual, undo_index;
  };
  std::vector<SOp> ops;

  long long sweeps = 0, scenarios = 0, topk_sweeps = 0, simulations = 0;
  double t_vq_copy = 0, t_vq_top = 0, t_prep_split[3] = {0, 0, 0};
  long long n_vq_copy = 0, n_vq_build = 0;
  double t_sweeps = 0, t_sim_setup = 0, t_evict = 0, t_victims_queue = 0, t_vq_pop = 0, t_tte = 0, t_addp = 0, t_filter = 0, t_bypod = 0, t_finit = 0;

  Solver(HostBackend &hb_, SolverScratch &scratch, std::vector<int> &n1, std::vector<int> &s1,
         std::vector<std::array<int, 3>> &extra)
      : hb(hb_), seq(hb_.seq), ctl(hb_.ctl), s(*hb_.seq.s), cfg(*hb_.seq.cfg), N(s.N), Q(s.Q), J(s.J), S(s.S), T(s.T),
        R(s.R), scr(scratch), on_node1(n1), on_status1(s1), on_extra(extra) {
    st = seq.rp.t_status;
    tn = seq.rp.t_node;
    tvirt = seq.rp.t_virtual;
    qa = seq.rp.q_alloc;
    qnp = seq.rp.q_alloc_np;
    scr.size_for(N, J, T);
    SolverScratch::bump(scr.slot_epoch, scr.slot_stamp);
    scr.slot_list.clear();
    setup_check = getenv("KAI_SOLVER_SETUP_CHECK") != nullptr;
    // Host answers need the mirror of every node and no topology term; with several GPUs every rank would answer alike,
    // but the multi-GPU path keeps its MINMAX exchange (DESIGN.md §7).
    const char *mx = getenv("KAI_HOST_SWEEP_MAX");
    host_sweep_max = mx ? atoi(mx) : kHostSweepMaxDefault;
    if (cfg.shard_count > 1 || seq.topology || !seq.mirror) host_sweep_max = 0;
    host_sweep_check = getenv("KAI_HOST_SWEEP_CHECK") != nullptr;
  }

  // ---------------- small accessors ----------------
  double req(int t, int r) const { return s.t_req[(size_t)t * R + r]; }
  int tjob(int t) const { return s.t_job[t]; }
  int ps_begin(int j) const { return s.j_ps_begin[j]; }
  int ps_end(int j) const { return s.j_ps_begin[j + 1]; }
  int pst_begin(int ps) const { return s.ps_task_begin[ps]; }
  int pst_end(int ps) const { return s.ps_task_begin[ps + 1]; }
  bool preemptible(int j) const { return (s.j_flags[j] & KAI_JOB_PREEMPTIBLE) != 0; }
  double &QA(int r, int q) { return qa[(size_t)r * Q + q]; }
  double &QNP(int r, int q) { return qnp[(size_t)r * Q + q]; }
  double qfair(int r, int q) const { return s.q_fair[(size_t)r * Q + q]; }
  double qdes(int r, int q) const { return s.q_deserved[(size_t)r * Q + q]; }
  double qlim(int r, int q) const { return s.q_limit[(size_t)r * Q + q]; }
  double qallocatable(int r, int q) const { return s.q_allocatable[(size_t)r * Q + q]; }
  bool should_allocate(int t, bool real) const {
    return st[t] == KAI_POD_PENDING || (!real && st[t] == KAI_POD_RELEASING && tvirt[t]);
  }
  int count_ps(int ps, int mask) const {
    if (mask == kActiveAllocated) return ps_active[ps];
    int c = 0;
    for (int t = pst_begin(ps); t < pst_end(ps); t++)
      if (st[t] & mask) c++;
    return c;
  }
  int count_job(int j, int mask) const {
    int c = 0;
    for (int ps = ps_begin(j); ps < ps_end(j); ps++) c += count_ps(ps, mask);
    return c;
  }
  bool job_ready(int j) const {  // subgroup_info/podset.go:114-120
    for (int ps = ps_begin(j); ps < ps_end(j); ps++)
      if (count_ps(ps, kAlive) - count_ps(ps, KAI_POD_GATED) < s.ps_min[ps]) return false;
    return true;
  }

  // ---------------- views: the session's jobs (id < J) and CloneWithTasks clones (job_info.go:477-510) ----------------
  // A clone owns copies of the PodSets: per-podset counters, Allocated and the inner caches are frozen at clone
  // time; the statuses of the tasks it lists stay live (the statement mutates the very PodInfo objects).
  typedef SolverJobCache Cache;
  struct View {
    int job = -1;
    std::vector<std::vector<int>> ps_tasks;
    std::vector<int> ps_min, ps_active_alloc;
    int active_alloc_total = 0, n_pending = 0;
    double allocated[QR] = {0, 0, 0};
    Cache cache;
  };
  std::vector<View> views;
  int vjob(int v) const { return v < J ? v : views[v - J].job; }
  Cache &vcache(int v) {  // live jobs (scr.job_cache): invalidated per action and on every status change (job_info.go:281-284)
    if (v >= J) return views[v - J].cache;
    Cache &c = scr.job_cache[v];
    if (c.stamp != scr.job_epoch) {
      c.stamp = scr.job_epoch;
      c.tta_valid = c.res_valid = false;
    }
    return c;
  }
  int v_nps(int v) const { return ps_end(vjob(v)) - ps_begin(vjob(v)); }
  int v_min(int v, int k) const { return v < J ? s.ps_min[ps_begin(v) + k] : views[v - J].ps_min[k]; }
  int v_active_alloc(int v, int k) const {
    return v < J ? count_ps(ps_begin(v) + k, kActiveAllocated) : views[v - J].ps_active_alloc[k];
  }
  std::vector<int> v_ps_tasks(int v, int k) const {
    if (v >= J) return views[v - J].ps_tasks[k];
    std::vector<int> out;
    int ps = ps_begin(v) + k;
    for (int t = pst_begin(ps); t < pst_end(ps); t++) out.push_back(t);
    return out;
  }
  std::vector<int> v_all_tasks(int v) const {
    std::vector<int> out;
    for (int k = 0; k < v_nps(v); k++)
      for (int t : v_ps_tasks(v, k)) out.push_back(t);
    return out;
  }
  int v_active_alloc_total(int v) const { return v < J ? count_job(v, kActiveAllocated) : views[v - J].active_alloc_total; }
  int v_pending(int v) const { return v < J ? count_job(v, KAI_POD_PENDING) : views[v - J].n_pending; }
  void v_allocated(int v, double *out) const {  // PodGroupInfo.Allocated (job_info.go:245-250)
    if (v >= J) {
      for (int r = 0; r < QR; r++) out[r] += views[v - J].allocated[r];
      return;
    }
    for (int ps = ps_begin(v); ps < ps_end(v); ps++)
      for (int t = pst_begin(ps); t < pst_end(ps); t++)
        if (st[t] & kAllocatedStatuses)
          for (int r = 0; r < QR; r++) out[r] += req(t, r);
  }
  int make_clone(int base, const std::vector<int> &tasks) {
    View c;
    c.job = vjob(base);
    int n = v_nps(base);
    c.ps_tasks.assign(n, {});
    c.ps_min.resize(n);
    c.ps_active_alloc.assign(n, 0);
    for (int k = 0; k < n; k++) c.ps_min[k] = v_min(base, k);
    for (int t : tasks) {
      int k = s.t_podset[t] - ps_begin(c.job);
      c.ps_tasks[k].push_back(t);
      if (st[t] & kActiveAllocated) {
        c.ps_active_alloc[k]++;
        c.active_alloc_total++;
      }
      if (st[t] == KAI_POD_PENDING) c.n_pending++;
      if (st[t] & kAllocatedStatuses)
        for (int r = 0; r < QR; r++) c.allocated[r] += req(t, r);
    }
    for (auto &v : c.ps_tasks) std::sort(v.begin(), v.end());
    views.push_back(c);
    return J + (int)views.size() - 1;
  }

  // ---------------- podset / task selection (allocation_info.go, eviction_info.go, subgroup_order.go) ----------------
  bool podset_less(int v, int ka, int kb) const {
    int ln = v_active_alloc(v, ka), rn = v_active_alloc(v, kb);
    int lmin = v_min(v, ka), rmin = v_min(v, kb);
    bool lsat = ln >= lmin, rsat = rn >= rmin;
    if (!lsat && !rsat) return ka < kb;
    if (!lsat) return true;
    if (!rsat) return false;
    double lr = (double)ln / (double)lmin, rr = (double)rn / (double)rmin;
    if (lr < rr) return true;
    if (rr < lr) return false;
    return ka < kb;
  }
  std::vector<int> ordered_podsets(int v) const {
    std::vector<int> o(v_nps(v));
    for (int k = 0; k < (int)o.size(); k++) o[k] = k;
    std::sort(o.begin(), o.end(), [&](int a, int b) { return podset_less(v, a, b); });
    return o;
  }
  std::vector<int> tasks_to_allocate(int v, bool real) {  // :27-54 (cached: the first caller decides `real`)
    if (vcache(v).tta_valid) return vcache(v).tta;
    std::vector<int> out;
    int unsat = 0;
    for (int k = 0; k < v_nps(v); k++)
      if (v_active_alloc(v, k) < v_min(v, k)) unsat++;
    int max_sets = unsat > 0 ? unsat : 1, n_sets = 0;
    for (int k : ordered_podsets(v)) {
      if (n_sets >= max_sets) break;
      std::vector<int> cand;
      for (int t : v_ps_tasks(v, k))
        if (should_allocate(t, real)) cand.push_back(t);
      if (cand.empty()) continue;
      int n_alloc = v_active_alloc(v, k);
      int max_tasks = n_alloc >= v_min(v, k) ? std::min((int)cand.size(), 1) : v_min(v, k) - n_alloc;
      for (int i = 0; i < (int)cand.size() && i < max_tasks; i++) out.push_back(cand[i]);
      n_sets++;
    }
    Cache &c = vcache(v);
    c.tta = out;
    c.tta_valid = true;
    return out;
  }
  const double *tta_init_resource(int v, bool real) {  // :87-113
    if (vcache(v).res_valid) return vcache(v).res;
    double acc[QR] = {0, 0, 0};
    for (int t : tasks_to_allocate(v, real))
      if (should_allocate(t, real))
        for (int r = 0; r < QR; r++) acc[r] += req(t, r);
    Cache &c = vcache(v);
    for (int r = 0; r < QR; r++) c.res[r] = acc[r];
    c.res_valid = true;
    return c.res;
  }
  std::vector<int> tasks_to_evict(int v, bool &has_more) {  // eviction_info.go:13-90
    std::vector<int> sets(v_nps(v));
    for (int k = 0; k < (int)sets.size(); k++) sets[k] = k;
    std::sort(sets.begin(), sets.end(), [&](int a, int b) { return podset_less(v, b, a); });
    int max_sets = (int)sets.size();
    for (int k = 0; k < v_nps(v); k++)
      if (v_active_alloc(v, k) > v_min(v, k)) {
        max_sets = 1;
        break;
      }
    std::vector<int> out;
    int n_sets = 0;
    for (int k : sets) {
      if (n_sets >= max_sets) break;
      std::vector<int> cand;
      for (int t : v_ps_tasks(v, k))
        if (st[t] & kActiveAllocated) cand.push_back(t);
      std::reverse(cand.begin(), cand.end());  // reverse TaskOrderFn
      int n_alloc = v_active_alloc(v, k);
      int max_tasks = n_alloc > v_min(v, k) ? 1 : n_alloc;
      for (int i = 0; i < (int)cand.size() && i < max_tasks; i++) out.push_back(cand[i]);
      n_sets++;
    }
    has_more = (int)out.size() < v_active_alloc_total(v);
    return out;
  }

  // ---------------- node accounting: host mirror of the GPU column + deltas to the owning scanner ----------------
  void touch(int n) {
    if (scr.node_stamp[n] != scr.node_epoch) {
      scr.node_stamp[n] = scr.node_epoch;
      scr.start_ig[n] = Ig(n);
      scr.start_lg[n] = Lg(n);
    }
  }
  double start_Ig(int n) const { return scr.node_stamp[n] == scr.node_epoch ? scr.start_ig[n] : Ig(n); }
  double start_Lg(int n) const { return scr.node_stamp[n] == scr.node_epoch ? scr.start_lg[n] : Lg(n); }
  // slot 0 of task t: the snapshot's until the action first changes t (status, node or slots), then scr.n0 / scr.s0
  int node0(int t) const {
    if (scr.slot_stamp[t] == scr.slot_epoch) return scr.n0[t];
    return (st[t] & kActiveUsed) && tn[t] >= 0 ? tn[t] : -1;
  }
  void take_slot(int t) {  // before the first change of t: copy its snapshot slot and list t for the teardown
    if (scr.slot_stamp[t] == scr.slot_epoch) return;
    scr.slot_stamp[t] = scr.slot_epoch;
    scr.n0[t] = (st[t] & kActiveUsed) && tn[t] >= 0 ? tn[t] : -1;
    scr.s0[t] = s.t_node_status[t];
    scr.slot_list.push_back(t);
  }
  int find_on(int t, int n) const {  // 0 / 1 = slot, 2 + i = on_extra[i], -1 = the task has no entry on node n
    if (node0(t) == n) return 0;
    if (on_node1[t] == n) return 1;
    for (size_t i = 0; i < on_extra.size(); i++)
      if (on_extra[i][0] == t && on_extra[i][1] == n) return 2 + (int)i;
    return -1;
  }
  double free_ready = 0;  // Σ idle + releasing GPUs over ready nodes (utils/action.go:145-160), kept incrementally
  void node_delta(int t, int n, int code) {
    touch(n);
    const double before = Ig(n) + Lg(n);
    emit_delta(seq, n, code, t);  // also applies the delta to the mirror (seq.mirror)
    if (s.nflags[n] & KAI_NODE_READY) free_ready += (Ig(n) + Lg(n)) - before;
    if (host_sweep_max > 0) gpu_free_update(n);
  }
  // nodes with idle or releasing GPUs right now (the XB_SNAP_GPUFREE definition), kept as the mirror changes, so that an
  // attempt's base feasible set is a copy of a short list rather than a scan of every node
  std::vector<int> gpu_free_list, gpu_free_pos;
  void gpu_free_update(int n) {
    const bool in = Ig(n) > 0 || Lg(n) > 0;
    if (in == (gpu_free_pos[n] >= 0)) return;
    if (in) {
      gpu_free_pos[n] = (int)gpu_free_list.size();
      gpu_free_list.push_back(n);
    } else {
      const int i = gpu_free_pos[n], last = gpu_free_list.back();
      gpu_free_list[i] = last;
      gpu_free_pos[last] = i;
      gpu_free_list.pop_back();
      gpu_free_pos[n] = -1;
    }
  }
  void node_add_task(int t) {  // node_info.go:457-493 with the task's current status
    take_slot(t);
    int n = tn[t], status = st[t];
    int e = find_on(t, n);
    if (e < 0) e = scr.n0[t] < 0 ? 0 : (on_node1[t] < 0 ? 1 : 2 + (int)on_extra.size());
    if (e >= 2) {
      if (e - 2 == (int)on_extra.size()) on_extra.push_back({t, n, status});
      on_extra[e - 2][2] = status;
    } else {
      (e == 0 ? scr.n0 : on_node1)[t] = n;
      (e == 0 ? scr.s0 : on_status1)[t] = status;
    }
    node_delta(t, n, status == KAI_POD_RELEASING ? ND_ADD_RELEASING : (status == KAI_POD_PIPELINED ? ND_ADD_PIPELINED : ND_ADD));
  }
  void node_remove_task(int t, int n) {  // :515-551 with the status of the clone stored on the node
    take_slot(t);
    int e = find_on(t, n);
    if (e < 0) return;  // node_info.go:495-501: a pod that is no longer on the node is an error, the node is untouched
    int status = e >= 2 ? on_extra[e - 2][2] : (e == 0 ? scr.s0 : on_status1)[t];
    node_delta(t, n, status == KAI_POD_RELEASING ? ND_REM_RELEASING : (status == KAI_POD_PIPELINED ? ND_REM_PIPELINED : ND_REM));
    if (e >= 2)
      on_extra.erase(on_extra.begin() + (e - 2));
    else
      (e == 0 ? scr.n0 : on_node1)[t] = -1;
  }
  // jobs with Pending tasks (utils.GetAllPendingJobs, actions/utils/action.go:122-130), kept as statuses change
  std::vector<int> pending_cnt;
  std::set<int> pending_jobs;
  // tasks with an active-allocated status per podset (count_ps(ps, kActiveAllocated)), kept by set_status: the
  // victims queues ask it of every job of every leaf queue
  std::vector<int> ps_active;
  void set_status(int t, int status) {
    take_slot(t);
    const int j = tjob(t);
    if (st[t] == KAI_POD_PENDING && status != KAI_POD_PENDING) {
      if (--pending_cnt[j] == 0) pending_jobs.erase(j);
    } else if (st[t] != KAI_POD_PENDING && status == KAI_POD_PENDING) {
      if (pending_cnt[j]++ == 0) pending_jobs.insert(j);
    }
    const bool was_active = (st[t] & kActiveAllocated) != 0, is_active = (status & kActiveAllocated) != 0;
    if (was_active != is_active) ps_active[s.t_podset[t]] += is_active ? 1 : -1;
    st[t] = status;
    Cache &c = vcache(j);
    c.tta_valid = c.res_valid = false;
    if (s.j_queue[j] >= 0) leaf_epoch[s.j_queue[j]]++;
  }
  void queue_allocate(int t, bool add) {  // proportion.go:443-489
    int j = tjob(t);
    bool np = !preemptible(j);
    for (int q = s.j_queue[j]; q >= 0; q = s.q_parent[q])
      for (int r = 0; r < QR; r++) {
        if (add) {
          QA(r, q) += req(t, r);
          if (np) QNP(r, q) += req(t, r);
        } else {
          QA(r, q) -= req(t, r);
          if (np) QNP(r, q) -= req(t, r);
        }
      }
  }

  // ---------------- Statement with undo chains (framework/statement.go) ----------------
  void stmt_pipeline(int t, int n, bool update_if_exists) {  // :197-295
    bool found = find_on(t, n) >= 0;
    if (found && !update_if_exists) {
      stmt_unevict(t);
      return;
    }
    SOp op{OPK_PIPELINE, t, st[t], tn[t], n, tvirt[t], -1};
    set_status(t, KAI_POD_PIPELINED);
    if (found) node_remove_task(t, n);
    tn[t] = n;
    node_add_task(t);
    queue_allocate(t, true);
    ops_push(op);
    tvirt[t] = 1;
  }
  void unpipeline(const SOp &op) {  // :432-476
    int t = op.task;
    set_status(t, op.prev_status);
    int host = tn[t];
    tn[t] = op.prev_node;
    tvirt[t] = (unsigned char)op.prev_virtual;
    node_remove_task(t, host);
    queue_allocate(t, false);
  }
  void stmt_evict(int t) {  // :63-128
    SOp op{OPK_EVICT, t, st[t], tn[t], tn[t], tvirt[t], -1};
    set_status(t, KAI_POD_RELEASING);
    node_remove_task(t, tn[t]);
    node_add_task(t);
    queue_allocate(t, false);
    ops_push(op);
    tvirt[t] = 1;
  }
  void unevict(const SOp &op) {  // :156-195
    int t = op.task;
    set_status(t, op.prev_status);
    tvirt[t] = (unsigned char)op.prev_virtual;
    int keep = tn[t];
    tn[t] = op.prev_node;
    node_remove_task(t, op.prev_node);
    node_add_task(t);
    tn[t] = keep;
    queue_allocate(t, true);
  }
  // :652-663 operationValid: decided by the FIRST undo operation that targets i (statement.go scans from the start
  // and returns at the first match), kept here as an index instead of a scan
  std::vector<int> first_undo;
  bool op_valid(int i) const {
    int u = i < (int)first_undo.size() ? first_undo[i] : -1;
    return u < 0 ? true : !op_valid(u);
  }
  void ops_push(const SOp &op) {
    ops.push_back(op);
    first_undo.push_back(-1);
    if (op.kind == OPK_UNDO && first_undo[op.undo_index] < 0) first_undo[op.undo_index] = (int)ops.size() - 1;
  }
  void ops_truncate(int n) {
    for (int u = (int)ops.size() - 1; u >= n; u--)
      if (ops[u].kind == OPK_UNDO && ops[u].undo_index < n && first_undo[ops[u].undo_index] == u) first_undo[ops[u].undo_index] = -1;
    ops.resize(n);
    first_undo.resize(n);
  }
  void undo_operation(int index) {  // :597-643
    if (!op_valid(index)) return;
    SOp op = ops[index];
    switch (op.kind) {
      case OPK_EVICT: unevict(op); break;
      case OPK_PIPELINE: unpipeline(op); break;
      case OPK_UNDO: redo_operation(op.undo_index); break;
      default: break;
    }
    ops_push(SOp{OPK_UNDO, -1, 0, -1, -1, 0, index});
  }
  void redo_operation(int index) {
    SOp op = ops[index];
    switch (op.kind) {
      case OPK_EVICT: stmt_evict(op.task); break;
      case OPK_PIPELINE: stmt_pipeline(op.task, op.next_node, true); break;
      case OPK_UNDO: undo_operation(op.undo_index); break;
      default: break;
    }
  }
  void stmt_unevict(int t) {  // :478-481 -> undoEarliestValidOperation
    for (int i = 0; i < (int)ops.size(); i++) {
      if (!op_valid(i)) continue;
      if (ops[i].kind != OPK_EVICT || ops[i].task != t) continue;
      undo_operation(i);
      return;
    }
  }
  int stmt_checkpoint() const { return (int)ops.size(); }
  void stmt_rollback(int cp) {
    for (int i = (int)ops.size() - 1; i >= cp; i--) undo_operation(i);
    ops_truncate(cp);
  }
  void stmt_discard() {
    for (int i = (int)ops.size() - 1; i >= 0; i--) undo_operation(i);
    ops_truncate(0);
  }
  void stmt_commit() {  // :536-571: pipelines keep Pipelined, evictions keep Releasing and stop being virtual
    commit_epoch++;
    for (int i = 0; i < (int)ops.size(); i++) {
      if (!op_valid(i)) continue;
      if (ops[i].kind == OPK_PIPELINE)
        seq.pods_placed++;
      else if (ops[i].kind == OPK_EVICT) {
        seq.pods_evicted++;
        tvirt[ops[i].task] = 0;
      }
    }
    ops_truncate(0);
  }

  // ---------------- capacity policy (proportion/capacity_policy) ----------------
  bool over_capacity(int j, const double *rq) {
    for (int q = s.j_queue[j]; q >= 0; q = s.q_parent[q])
      for (int r = 0; r < QR; r++) {
        if (qlim(r, q) == KAI_UNLIMITED || rq[r] == 0) continue;
        if (qlim(r, q) < QA(r, q) + rq[r]) return true;
      }
    if (preemptible(j)) return false;
    for (int q = s.j_queue[j]; q >= 0; q = s.q_parent[q])
      for (int r = 0; r < QR; r++) {
        if (qdes(r, q) == KAI_UNLIMITED || rq[r] == 0) continue;
        if (qdes(r, q) < QNP(r, q) + rq[r]) return true;
      }
    return false;
  }

  // ---------------- GPU sweeps ----------------
  bool gpu_failed() const { return hb.failed || seq.error == kSeqErrHostSweep; }
  // allocateTask (allocate.go:121-163) in a simulation: one restricted pipeline-only sweep
  unsigned int sweep_extra_bits = 0;  // XB_RESTRICT_DOM while a topology domain is selected
  int sweep_pick_node(int t) {
    Decision &d = ctl.dec;
    for (int r = 0; r < KAI_MAX_RES; r++) d.req[r] = r < R ? req(t, r) : 0.0;
    d.gpu_task = d.req[KAI_RES_GPU] > 0;
    d.res = d.gpu_task ? KAI_RES_GPU : KAI_RES_CPU;
    d.strategy = d.gpu_task ? cfg.gpu_placement : cfg.cpu_placement;
    d.pipeline_only = 1;
    d.nominated = s.t_nominated ? s.t_nominated[t] : -1;
    d.pred_class = s.t_pred_class ? s.t_pred_class[t] : -1;
    bool empty = !(d.req[KAI_RES_GPU] > 0.01) && !(d.req[KAI_RES_CPU] >= 10) && !(d.req[KAI_RES_MEM] >= 10.0 * 1024 * 1024);
    for (int r = 3; r < R; r++)
      if (d.req[r] >= 10) empty = false;
    d.best_effort = empty;
    d.restricted = 1;
    d.task = t;
    ctl.batch.valid = 0;
    // pack.go:66-86 over the node set of this simulation: the scanners exchange their extremes among themselves
    ctl.trk[0].dirty = ctl.trk[1].dirty = 1;
    const double t0 = HostBackend::now();
    const bool on_host = host_sweep_usable();
    if (!on_host || host_sweep_check) {
      hb.sweep_single(sweep_extra_bits);  // only the winner is needed
      sweeps++;
    }
    if (on_host && !hb.failed) {
      const Winner w = host_sweep();
      if (host_sweep_check && !same_winner(w, ctl.win)) {
        snprintf(hb.error_msg, sizeof(hb.error_msg),
                 "KAI_HOST_SWEEP_CHECK: task %d: host sweep picked node %d (score bits %016llx, rank %u, flags %u), "
                 "GPU sweep node %d (score bits %016llx, rank %u, flags %u)",
                 t, w.node, (unsigned long long)kbits(w.score), w.rank, w.flags, ctl.win.node,
                 (unsigned long long)kbits(ctl.win.score), ctl.win.rank, ctl.win.flags);
        seq.error = kSeqErrHostSweep;
      }
      ctl.win = w;
      host_sweeps++;
    }
    t_sweeps += HostBackend::now() - t0;
    if (gpu_failed()) return -1;
    return ctl.win.node;
  }
  // ---- restricted sweeps answered from the host mirror ----
  // A simulation's feasible set (FeasibleNodesForJob) is the attempt's base set (nodes with idle or releasing GPUs when
  // the attempt started) plus the victims' nodes.  When it holds at most host_sweep_max rows, the answer is computed here
  // from seq.mirror in the scanners' order (extremes, predicate mask, node_key, argmax on score desc / name rank asc)
  // instead of a GPU round trip.  No record is published: the queued node and feasible-set deltas stay queued for the
  // next record, so the scanners' tiles stay in step, and no sequence number is consumed.
  static constexpr int kHostSweepMaxDefault = 256;
  static constexpr int kSeqErrHostSweep = 3;  // Seq::error: KAI_HOST_SWEEP_CHECK or KAI_SOLVER_SETUP_CHECK found a difference
  int host_sweep_max = 0;         // KAI_HOST_SWEEP_MAX (0: every sweep runs on the GPU)
  bool host_sweep_check = false;  // KAI_HOST_SWEEP_CHECK: run the GPU sweep as well and fail on any difference
  long long host_sweeps = 0;
  std::vector<int> base_list;  // the attempt's base feasible set (valid when base_known)
  bool base_known = false;
  bool host_sweep_usable() const {
    return host_sweep_max > 0 && base_known && !feas_all && sweep_extra_bits == 0 &&
           base_list.size() + feas_extra_list.size() <= (size_t)host_sweep_max;
  }
  static bool same_winner(const Winner &a, const Winner &b) {
    return a.node == b.node && a.rank == b.rank && a.flags == b.flags && (a.node < 0 || kbits(a.score) == kbits(b.score));
  }
  Winner host_sweep() {
    Decision d = ctl.dec;
    const double *Ag = s.alloc + (size_t)KAI_RES_GPU * N, *Ac = s.alloc + (size_t)KAI_RES_CPU * N;
    const int nb = (int)base_list.size(), ne = (int)feas_extra_list.size();
    auto row_at = [&](int i) { return i < nb ? base_list[i] : feas_extra_list[i - nb]; };
    if (d.strategy == KAI_PLACEMENT_BINPACK) {  // the fused min/max of the scanners (XB_FUSED_MM)
      double mn = DBL_MAX, mx = 0;
      const double *A = d.res == KAI_RES_GPU ? Ag : Ac;
      for (int i = 0; i < nb + ne; i++) {
        const int n = row_at(i);
        if (A[n] == 0) continue;
        const double *row = seq.mirror + (size_t)n * 2 * R;
        const double cur = kadd(row[d.res], row[R + d.res]);
        if (cur < mn) mn = cur;
        if (cur > mx) mx = cur;
      }
      d.mn = mn;
      d.mx = mx;
    }
    const uint32_t *mask = d.pred_class >= 0 ? s.pred_mask + (size_t)d.pred_class * s.mask_words : nullptr;
    double bs = -1.0;
    uint32_t brank = kRankNone;
    int bnode = -1;
    bool bfit_i = false;
    for (int i = 0; i < nb + ne; i++) {
      const int n = row_at(i);
      if (mask && !((mask[n >> 5] >> (n & 31)) & 1u)) continue;
      const double *row = seq.mirror + (size_t)n * 2 * R;
      double score;
      bool fit_i;
      if (!node_key(d, R, row, row + R, 1, Ag[n], Ac[n], s.gpu_count[n], s.nflags[n], n, score, fit_i)) continue;
      const uint32_t rk = (uint32_t)s.name_rank[n];
      if (better(score, rk, bs, brank)) {
        bs = score;
        brank = rk;
        bnode = n;
        bfit_i = fit_i;
      }
    }
    Winner w;
    w.score = bs;
    w.rank = brank;
    w.node = bnode;
    // publish_candidate's flags; the trackers are dirty (no event bits) and nothing is batched
    w.flags = (bnode >= 0 && !d.pipeline_only && (d.best_effort || bfit_i)) ? SLOT_TO_IDLE : 0u;
    return w;
  }
  // the k rows with most idle + releasing GPUs (values, descending); pages of top-M lists until k are known
  std::vector<std::pair<double, int>> sweep_topk_idle(int k, unsigned int snap_bits) {
    std::vector<std::pair<double, int>> host;
    const bool on_host = host_sweep_max > 0 && host_topk(k, host);
    if (on_host && !host_sweep_check) {
      if (snap_bits) {  // the feasible-set snapshot still reaches the scanners, without a round trip
        ctl.xbits = snap_bits;
        hb.flush_deltas();
        ctl.xbits = 0;
      }
      host_topks++;
      return host;
    }
    std::vector<std::pair<double, int>> dev = sweep_topk_idle_gpu(k, snap_bits);
    // KAI_HOST_SWEEP_CHECK: every answer, the GPU's list and the host one, against the plain restatement over all rows
    // (one GPU: a shard's mirror holds every row, but its list only its own)
    if (host_sweep_check && seq.mirror && cfg.shard_count <= 1 && !hb.failed) {
      const std::vector<std::pair<double, int>> ref = topk_reference(k);
      if (on_host) topk_check("host", k, host, ref);
      topk_check("GPU", k, dev, ref);
    }
    if (on_host) {
      host_topks++;
      return host;
    }
    return dev;
  }
  // The k rows with most idle + releasing GPUs, restated: every mirror row, key = Idle + Releasing GPUs, sorted by key
  // descending and name rank ascending (-0.0 == +0.0, so the rank decides between them).
  std::vector<std::pair<double, int>> topk_reference(int k) const {
    std::vector<int> rows(N);
    for (int n = 0; n < N; n++) rows[n] = n;
    const size_t m = std::min((size_t)std::max(k, 0), (size_t)N);
    auto key = [&](int n) { return kadd(Ig(n), Lg(n)); };
    std::partial_sort(rows.begin(), rows.begin() + m, rows.end(), [&](int a, int b) {
      const double ka = key(a), kb = key(b);
      return ka > kb || (ka == kb && s.name_rank[a] < s.name_rank[b]);
    });
    std::vector<std::pair<double, int>> out;
    for (size_t i = 0; i < m; i++) out.push_back({key(rows[i]), rows[i]});
    return out;
  }
  void topk_check(const char *who, int k, const std::vector<std::pair<double, int>> &got,
                  const std::vector<std::pair<double, int>> &ref) {
    if (seq.error == kSeqErrHostSweep) return;  // the first difference is the one reported
    size_t i = 0;
    while (i < got.size() && i < ref.size() && got[i] == ref[i]) i++;  // pair ==: values compare as doubles
    if (i == got.size() && i == ref.size()) return;
    snprintf(hb.error_msg, sizeof(hb.error_msg),
             "KAI_HOST_SWEEP_CHECK: top-%d idle-GPU rows differ: %s %zu rows, reference %zu rows; first difference at "
             "%zu: %s node %d (%g), reference node %d (%g)",
             k, who, got.size(), ref.size(), i, who, i < got.size() ? got[i].second : -1, i < got.size() ? got[i].first : 0.0,
             i < ref.size() ? ref[i].second : -1, i < ref.size() ? ref[i].first : 0.0);
    seq.error = kSeqErrHostSweep;
  }
  // The same k rows from the mirror: every row with idle + releasing GPUs > 0 is in gpu_free_list; after them come the
  // rows whose sum is exactly 0, in name-rank order (rows below 0 would follow: the GPU answers when they are needed).
  long long host_topks = 0;
  bool host_topk(int k, std::vector<std::pair<double, int>> &out) {
    if (gpu_free_list.size() > (size_t)host_sweep_max) return false;
    struct Row {
      double key;
      int rank, node;
    };
    std::vector<Row> pos;
    for (int n : gpu_free_list) {
      const double key = kadd(Ig(n), Lg(n));
      if (key > 0) pos.push_back({key, s.name_rank[n], n});
    }
    std::sort(pos.begin(), pos.end(), [](const Row &a, const Row &b) { return a.key > b.key || (a.key == b.key && a.rank < b.rank); });
    out.clear();
    for (size_t i = 0; i < pos.size() && (int)out.size() < k; i++) out.push_back({pos[i].key, pos[i].node});
    const int scan_cap = 4 * host_sweep_max + k;
    for (int r = 0; r < N && (int)out.size() < k; r++) {
      if (r >= scan_cap) return false;
      const int n = hb.rank_to_node[r];
      const double key = kadd(Ig(n), Lg(n));
      if (key == 0) out.push_back({key, n});
    }
    return (int)out.size() == std::min(k, N);
  }
  std::vector<std::pair<double, int>> sweep_topk_idle_gpu(int k, unsigned int snap_bits) {
    std::vector<std::pair<double, int>> out;
    Decision &d = ctl.dec;
    d.restricted = 0;
    double cut_key = 0, cut_rank = 0, has_cut = 0;
    for (;;) {
      for (int r = 0; r < KAI_MAX_RES; r++) d.req[r] = 0;
      d.req[0] = cut_key;
      d.req[1] = cut_rank;
      d.req[2] = has_cut;
      ctl.xbits = snap_bits;
      snap_bits = 0;
      hb.publish(DK_TOPK);
      ctl.xbits = 0;
      hb.gather_list();
      topk_sweeps++;
      if (hb.failed) break;
      for (size_t i = 0; i < hb.list_valid && (int)out.size() < k; i++) out.push_back({hb.list[i].score, hb.list[i].node});
      if ((int)out.size() >= k || hb.list_valid == 0 || !hb.list_more) break;
      const HostBackend::ListCand &last = hb.list[hb.list_valid - 1];
      cut_key = last.score;
      cut_rank = (double)last.rank;
      has_cut = 1;
    }
    hb.list_invalidate();
    return out;
  }

  // session side of TopoAllocator for simulations: views with frozen counters, the solver's statement, the feasible set
  struct SimOps {
    Solver &so;
    int v;
    int k_of(int ps) const { return ps - so.ps_begin(so.vjob(v)); }
    int active_alloc(int ps) { return so.v_active_alloc(v, k_of(ps)); }
    void active_nodes(int ps, std::vector<int> &out) {
      for (int t : so.v_ps_tasks(v, k_of(ps)))
        if (so.st[t] & kActiveAllocated) out.push_back(so.tn[t]);
    }
    bool podset_less(int a, int b) { return so.podset_less(v, k_of(a), k_of(b)); }
    int checkpoint() { return so.stmt_checkpoint(); }
    void rollback(int cp) { so.stmt_rollback(cp); }
    bool place(const std::vector<int> &tasks, unsigned int xbits) {
      so.sweep_extra_bits = xbits;
      bool ok = true;
      for (int t : tasks)
        if (!so.allocate_task(t)) {
          ok = false;
          break;
        }
      so.sweep_extra_bits = 0;
      return ok && !so.gpu_failed();
    }
    bool extra_in_set(int n) { return so.in_base(n) || so.feas_extra[n]; }
    bool all_nodes() { return false; }
  };
  // ---------------- actions/common/allocate.go on views, pipeline-only ----------------
  const std::vector<char> *feasible = nullptr;
  bool allocate_task(int t) {
    double creq[QR] = {req(t, KAI_RES_CPU), req(t, KAI_RES_MEM), req(t, KAI_RES_GPU) > 0 ? 1.0 : 0.0};
    if (over_capacity(tjob(t), creq)) return false;
    int n = sweep_pick_node(t);
    if (n < 0) return false;
    stmt_pipeline(t, n, false);
    return true;
  }
  bool allocate_job(int v) {
    std::vector<int> tta = tasks_to_allocate(v, false);
    int j = vjob(v);
    double rq[QR] = {0, 0, 0};
    for (int t : tta)
      for (int r = 0; r < QR; r++) rq[r] += req(t, r);
    if (over_capacity(j, rq)) return false;
    TopologyHost *topo = (TopologyHost *)seq.topology;
    if (topo && topo->constrained(j)) {  // SubGroupSet tree / topology constraints: allocate.go:36-83 via TopoAllocator
      SimOps ops{*this, v};
      TopoAllocator<SimOps> ta(*topo, seq, ops, j);
      bool placed = ta.alloc_set(topo->job_root_set[j], tta);
      if (ta.unsupported) seq.error = 2;
      sweep_extra_bits = 0;
      return placed;
    }
    if (topo) topo->scores_off(seq);
    int cp = stmt_checkpoint();
    for (int k : ordered_podsets(v)) {
      int ps = ps_begin(j) + k;
      int cp2 = stmt_checkpoint();
      bool ok = true;
      for (int t : tta) {
        if (s.t_podset[t] != ps) continue;
        if (!allocate_task(t)) {
          ok = false;
          break;
        }
      }
      if (!ok) {
        stmt_rollback(cp2);
        stmt_rollback(cp);
        return false;
      }
    }
    return true;
  }

  // ---------------- queue order (proportion/queue_order/queue_order.go:19-273) ----------------
  double dominant_share(int q, const double *alloc) const {  // queue_resource_share.go:142-166
    double m = 0;
    for (int r = 0; r < QR; r++) {
      double la = qallocatable(r, q);
      double denom = la == KAI_UNLIMITED ? s.total[r] : la;
      double v = denom == 0 ? alloc[r] * 1000.0 : alloc[r] / denom;
      m = std::max(m, v);
    }
    return m;
  }
  int queue_order_result(int l, int r, const double *lreq, const double *rreq, const double *lvict, const double *rvict) {
    bool lover = true, rover = true;
    for (int i = 0; i < QR; i++) {
      if (qfair(i, l) >= QA(i, l)) lover = false;
      if (qfair(i, r) >= QA(i, r)) rover = false;
    }
    if (!lover && rover) return -1;
    if (lover && !rover) return 1;
    double lw[QR], rw[QR];
    for (int i = 0; i < QR; i++) {
      lw[i] = QA(i, l) + lreq[i];
      rw[i] = QA(i, r) + rreq[i];
    }
    bool lst = true, rst = true;
    for (int i = 0; i < QR; i++) {
      if (compare_quantities(lw[i], qdes(i, l)) > 0) lst = false;
      if (compare_quantities(rw[i], qdes(i, r)) > 0) rst = false;
    }
    if (lst && !rst) return -1;
    if (rst && !lst) return 1;
    if (s.q_priority[l] > s.q_priority[r]) return -1;
    if (s.q_priority[l] < s.q_priority[r]) return 1;
    bool lv = false, rv = false;
    for (int i = 0; i < QR; i++) {
      if (qallocatable(i, l) == 0 && lw[i] > 0) lv = true;
      if (qallocatable(i, r) == 0 && rw[i] > 0) rv = true;
    }
    if (lv && !rv) return 1;
    if (!lv && rv) return -1;
    double la[QR], ra[QR];
    for (int i = 0; i < QR; i++) {
      la[i] = QA(i, l) + lreq[i];
      ra[i] = QA(i, r) + rreq[i];
      if (lvict) la[i] -= lvict[i];
      if (rvict) ra[i] -= rvict[i];
    }
    double ls = dominant_share(l, la), rs = dominant_share(r, ra);
    if (ls < rs) return -1;
    if (ls > rs) return 1;
    double lcur[QR], rcur[QR];
    for (int i = 0; i < QR; i++) {
      lcur[i] = QA(i, l);
      rcur[i] = QA(i, r);
    }
    ls = dominant_share(l, lcur);
    rs = dominant_share(r, rcur);
    if (ls < rs) return -1;
    if (ls > rs) return 1;
    bool l_le_r = true, r_le_l = true;
    for (int i = 0; i < QR; i++) {
      if (compare_quantities(qallocatable(i, l), qallocatable(i, r)) > 0) l_le_r = false;
      if (compare_quantities(qallocatable(i, r), qallocatable(i, l)) > 0) r_le_l = false;
    }
    if (!r_le_l && l_le_r) return -1;
    if (!l_le_r && r_le_l) return 1;
    return s.q_creation[l] < s.q_creation[r] ? -1 : 1;
  }

  // ---------------- JobsOrderByQueues (actions/utils/job_order_by_queue.go) over views ----------------
  // Flat form: every heap of the tree (root, queue nodes, leaves) is a range of one arena, nodes are plain data and the
  // comparators are small function objects over the owning JobsOrder, so a copy is a few contiguous copies and a build
  // allocates nothing per node.  A heap that outgrows its range moves to the end of the arena.
  struct HeapRange {
    int off = 0, len = 0, cap = 0;
  };
  struct QNode {
    int queue = -1, parent = -1;
    bool is_leaf = false, needs_reorder = false, linked = false;
    int lazy_queue = -1;  // victims queue: only the best job of this leaf is loaded so far (Solver::victim_leaf_list has the rest)
    HeapRange children;
  };
  struct JobsOrder;
  struct JobLess {  // leaf heaps: JobOrderFn, inverted for the victims queue
    const JobsOrder *jo;
    bool operator()(int a, int b) const { return jo->victim_queue ? !jo->job_less(a, b) : jo->job_less(a, b); }
  };
  struct NodeLess {  // root and queue-node heaps: QueueOrderFn
    JobsOrder *jo;
    bool operator()(int a, int b) const { return jo->node_less(a, b); }
  };
  struct JobsOrder {
    Solver *o = nullptr;
    bool victim_queue = false;
    std::vector<QNode> nodes;
    std::vector<int> queue_node;
    std::vector<int> arena;
    HeapRange root;
    std::vector<double> popped_alloc;  // [Q][3] running Allocated sum of the victims popped per queue (victims queue)

    int *heap_data(const HeapRange &h) { return arena.data() + h.off; }
    const int *heap_data(const HeapRange &h) const { return arena.data() + h.off; }
    int peek(const HeapRange &h) const { return arena[h.off]; }
    HeapRange &heap_of(int ni) { return ni < 0 ? root : nodes[ni].children; }  // ni = -1: the root heap
    bool heap_is_leaf(int ni) const { return ni >= 0 && nodes[ni].is_leaf; }
    void reserve_heap(int ni, int need) {  // room for `need` entries; moves the range to the end of the arena if short
      HeapRange &h = heap_of(ni);
      if (need <= h.cap) return;
      const int cap = std::max(need, 2 * h.cap), off = (int)arena.size();
      arena.resize((size_t)off + cap);
      std::copy(arena.begin() + h.off, arena.begin() + h.off + h.len, arena.begin() + off);
      h.off = off;
      h.cap = cap;
    }
    void heap_assign(int ni, const int *src, int n) {  // the entries as they are (a sorted run is already a heap)
      heap_of(ni).len = 0;
      reserve_heap(ni, n);
      HeapRange &h = heap_of(ni);
      std::copy(src, src + n, arena.begin() + h.off);
      h.len = n;
    }
    void heap_push(int ni, int x) {
      reserve_heap(ni, heap_of(ni).len + 1);
      HeapRange &h = heap_of(ni);
      if (heap_is_leaf(ni))
        HeapGo::push(heap_data(h), h.len, x, JobLess{this});
      else
        HeapGo::push(heap_data(h), h.len, x, NodeLess{this});
    }
    int heap_pop(int ni) {
      HeapRange &h = heap_of(ni);
      return heap_is_leaf(ni) ? HeapGo::pop(heap_data(h), h.len, JobLess{this}) : HeapGo::pop(heap_data(h), h.len, NodeLess{this});
    }
    void heap_fix(int ni, int i) {
      HeapRange &h = heap_of(ni);
      if (heap_is_leaf(ni))
        HeapGo::fix(heap_data(h), h.len, i, JobLess{this});
      else
        HeapGo::fix(heap_data(h), h.len, i, NodeLess{this});
    }

    void min_available_state(int v, bool &below, bool &above, bool &exactly) const {  // elastic.go:50-63
      exactly = true;
      for (int k = 0; k < o->v_nps(v); k++) {
        int n = o->v_active_alloc(v, k);
        if (n < o->v_min(v, k)) {
          below = true;
          above = false;
          exactly = false;
          return;
        }
        if (n > o->v_min(v, k)) exactly = false;
      }
      below = false;
      above = !exactly;
    }
    bool job_less(int l, int r) const {  // session_plugins.go:227-242
      int lj = o->vjob(l), rj = o->vjob(r);
      if (o->s.j_priority[lj] > o->s.j_priority[rj]) return true;
      if (o->s.j_priority[lj] < o->s.j_priority[rj]) return false;
      bool lb, la, le, rb, ra, re;
      min_available_state(l, lb, la, le);
      min_available_state(r, rb, ra, re);
      if (lb && !rb) return true;
      if (le && ra) return true;
      if (!lb && rb) return false;
      if (la && re) return false;
      return o->s.j_order_rank[lj] < o->s.j_order_rank[rj];
    }
    int best_job(int ni) const { return nodes[ni].is_leaf ? peek(nodes[ni].children) : best_job(peek(nodes[ni].children)); }
    int leaf_of_best(int ni) const { return nodes[ni].is_leaf ? ni : leaf_of_best(peek(nodes[ni].children)); }
    bool node_less(int l, int r) {  // :256-278
      if (nodes[l].children.len == 0) return !victim_queue;
      if (nodes[r].children.len == 0) return victim_queue;
      double lreq[QR] = {0, 0, 0}, rreq[QR] = {0, 0, 0}, lv[QR] = {0, 0, 0}, rv[QR] = {0, 0, 0};
      if (!victim_queue) {
        const double *a = o->tta_init_resource(best_job(l), false);
        for (int i = 0; i < QR; i++) lreq[i] = a[i];
        const double *b = o->tta_init_resource(best_job(r), false);
        for (int i = 0; i < QR; i++) rreq[i] = b[i];
      } else {
        victims_allocated(l, lv);
        victims_allocated(r, rv);
      }
      int res = o->queue_order_result(nodes[l].queue, nodes[r].queue, lreq, rreq, victim_queue ? lv : nullptr,
                                      victim_queue ? rv : nullptr);
      bool result = res < 0;
      return victim_queue ? !result : result;
    }
    void victims_allocated(int ni, double *out) {  // :338-346
      // Allocated of the victims popped from this queue so far + of its best remaining job, summed task by task in pop
      // order.  The popped part is kept as a running sum (the same left fold: each pop continues it), so a comparison
      // costs O(1) instead of O(victims popped) — with thousands of victims per queue the literal loop made the victims
      // queue quadratic (4.6 of 6.1 s of `reclaim` at cycle5-1000).  `out` arrives zeroed.
      int leaf = leaf_of_best(ni);
      const double *acc = popped_alloc.data() + (size_t)nodes[leaf].queue * QR;
      for (int r = 0; r < QR; r++) out[r] = acc[r];
      if (nodes[leaf].children.len != 0) o->v_allocated(peek(nodes[leaf].children), out);
    }
    void copy_from(const JobsOrder &src) {
      o = src.o;
      victim_queue = src.victim_queue;
      nodes = src.nodes;
      queue_node = src.queue_node;
      arena = src.arena;
      root = src.root;
      popped_alloc = src.popped_alloc;
    }
    void init(Solver *solver, bool victims) {
      o = solver;
      victim_queue = victims;
      nodes.clear();
      queue_node.assign(o->Q, -1);
      arena.clear();
      root = HeapRange();
      if (victims)
        popped_alloc.assign((size_t)o->Q * QR, 0.0);
      else
        popped_alloc.clear();
    }
    int make_node(int q, bool leaf) {  // a queue node's heap holds at most its child queues
      nodes.emplace_back();
      int id = (int)nodes.size() - 1;
      nodes[id].queue = q;
      nodes[id].is_leaf = leaf;
      reserve_heap(id, leaf ? 1 : std::max(1, o->s.q_nchildren[q]));
      return id;
    }
    void mark_ancestors(int ni) {
      for (int c = ni; c >= 0; c = nodes[c].parent) nodes[c].needs_reorder = true;
    }
    void ensure_chain(int child) {  // :135-175
      int cq = nodes[child].queue;
      if (o->s.q_parent[cq] < 0) {
        if (!nodes[child].linked) {
          heap_push(-1, child);
          nodes[child].linked = true;
        }
        return;
      }
      int pq = o->s.q_parent[cq];
      int pn = queue_node[pq];
      bool is_new = pn < 0;
      if (is_new) {
        pn = make_node(pq, false);
        queue_node[pq] = pn;
      }
      if (!nodes[child].linked) {
        nodes[child].parent = pn;
        heap_push(pn, child);
        nodes[child].linked = true;
      }
      if (is_new) ensure_chain(pn);
    }
    // a lazily loaded leaf holds its best job only; anything that reads or changes more loads the whole run first
    void materialize(int leaf) {
      if (nodes[leaf].lazy_queue < 0) return;
      const int q = nodes[leaf].lazy_queue;
      nodes[leaf].lazy_queue = -1;
      const std::vector<int> &run = o->victim_leaf_list(*this, q);  // same best job on top: the ancestors' heaps are unaffected
      heap_assign(leaf, run.data(), (int)run.size());
    }
    void push_job(int v) {  // :90-119
      int q = o->s.j_queue[o->vjob(v)];
      if (q < 0 || o->s.q_nchildren[q] != 0) return;
      int leaf = queue_node[q];
      if (leaf >= 0) materialize(leaf);
      bool needs_linking = leaf < 0;
      if (needs_linking) {
        leaf = make_node(q, true);
        queue_node[q] = leaf;
      }
      heap_push(leaf, v);
      if (needs_linking) ensure_chain(leaf);
      mark_ancestors(leaf);
    }
    bool is_empty() const { return root.len == 0; }
    int get_next_node(int hi) {  // :193-215 (hi: the heap's owner, -1 = root)
      for (;;) {
        const HeapRange &h = heap_of(hi);
        if (h.len == 0) return -1;
        int ni = peek(h);
        if (nodes[ni].needs_reorder) {
          heap_fix(hi, 0);
          nodes[ni].needs_reorder = false;
          continue;
        }
        if (nodes[ni].children.len == 0) return -1;
        return ni;
      }
    }
    void handle_pop(int ni) {  // :219-243
      if (nodes[ni].children.len == 0) {
        heap_pop(nodes[ni].parent);  // parent -1: the root heap
        queue_node[nodes[ni].queue] = -1;
        nodes[ni].linked = false;
        if (nodes[ni].parent >= 0) handle_pop(nodes[ni].parent);
        return;
      }
      mark_ancestors(ni);
    }
    int pop_next_job() {  // :61-88
      if (is_empty()) return -1;
      int hi = -1;
      int leaf = -1;
      for (;;) {
        int ni = get_next_node(hi);
        if (ni < 0) return -1;
        if (nodes[ni].is_leaf) {
          leaf = ni;
          break;
        }
        hi = ni;
      }
      materialize(leaf);
      int job = heap_pop(leaf);
      if (victim_queue) o->v_allocated(job, popped_alloc.data() + (size_t)nodes[leaf].queue * QR);
      handle_pop(leaf);
      return job;
    }
  };
  struct OrderOpts {
    bool filter_unready = false, filter_non_pending = false, filter_non_preemptible = false, filter_non_active_allocated = false;
  };
  // input_jobs.go:21-68; canonical order: leaf queues ascending, the jobs of a queue in the heap's own order
  void init_jobs_order(JobsOrder &jo, const std::vector<int> &vs, const OrderOpts &op) {
    std::vector<std::vector<int>> by_queue(Q);
    for (int v : vs) {
      int j = vjob(v);
      if (op.filter_unready && !job_ready(j)) continue;
      if (op.filter_non_pending && v_pending(v) == 0) continue;
      if (op.filter_non_preemptible && !preemptible(j)) continue;
      if (op.filter_non_active_allocated) {
        bool active = false;
        for (int t : v_all_tasks(v))
          if (st[t] & kActiveAllocated) active = true;
        if (!active) continue;
      }
      int q = s.j_queue[j];
      if (q < 0 || s.q_nchildren[q] != 0) continue;
      by_queue[q].push_back(v);
    }
    for (int q = 0; q < Q; q++) {
      std::sort(by_queue[q].begin(), by_queue[q].end(),
                [&](int a, int b) { return jo.victim_queue ? jo.job_less(b, a) : jo.job_less(a, b); });
      for (int v : by_queue[q]) jo.push_job(v);
    }
  }

  // ---------------- scenario (scenario/base_scenario.go, by_node_scenario.go) ----------------
  struct Scenario {
    int preemptor = -1;
    std::vector<int> pending_tasks, potential_tasks, recorded_jobs, recorded_tasks;
    std::map<int, std::vector<int>> victims, task_groups, jobs_by_node;
  };
  void scenario_append_group(Scenario &sc, const std::vector<int> &tasks) {
    int j = tjob(tasks[0]);
    sc.task_groups[j].push_back(make_clone(j, tasks));
    auto &vt = sc.victims[j];
    vt.insert(vt.end(), tasks.begin(), tasks.end());
  }
  void scenario_add_potential(Scenario &sc, const std::vector<int> &tasks) {
    if (tasks.empty()) return;
    sc.potential_tasks.insert(sc.potential_tasks.end(), tasks.begin(), tasks.end());
    scenario_append_group(sc, tasks);
    for (int t : tasks) {
      auto &v = sc.jobs_by_node[tn[t]];
      if (std::find(v.begin(), v.end(), tjob(t)) == v.end()) v.push_back(tjob(t));
    }
  }
  std::vector<int> scenario_victims_from_node(const Scenario &sc, int node) {
    std::vector<int> out;
    auto it = sc.jobs_by_node.find(node);
    if (it == sc.jobs_by_node.end()) return out;
    std::vector<int> jobs = it->second;
    std::sort(jobs.begin(), jobs.end());
    for (int j : jobs) {
      auto g = sc.task_groups.find(j);
      if (g == sc.task_groups.end()) continue;
      for (int group : g->second)
        for (int t : v_all_tasks(group)) out.push_back(t);
    }
    return out;
  }

  // ---------------- idle-GPU scenario filter (idle_gpus.go, common.go) ----------------
  struct IdleFilter {
    int k = 0;
    std::map<int, double> value;  // nodes of the base top-k and nodes that received victims' GPUs
    std::multiset<double, std::greater<double>> sorted;  // the same values, descending (incremental, like orderedInsert)
    size_t n_rec_done = 0, n_pot_done = 0;
    std::vector<double> rq;  // GPU requests of the pending tasks, descending
  };
  void idle_filter_account(IdleFilter &f, const Scenario &sc) {
    // recorded victims never change within a builder and potential victims are append-only: only new entries
    for (const std::vector<int> *lst : {&sc.recorded_tasks, &sc.potential_tasks})
      for (size_t i = (lst == &sc.recorded_tasks ? f.n_rec_done : f.n_pot_done); i < lst->size(); i++) {
        const int t = (*lst)[i];
        if (tn[t] < 0 || scr.seen_stamp[t] == scr.seen_epoch) continue;
        scr.seen_stamp[t] = scr.seen_epoch;
        auto it = f.value.find(tn[t]);
        if (it == f.value.end())
          it = f.value.emplace(tn[t], start_Ig(tn[t]) + start_Lg(tn[t])).first;
        else
          f.sorted.erase(f.sorted.find(it->second));
        it->second += req(t, KAI_RES_GPU);
        f.sorted.insert(it->second);
      }
    f.n_rec_done = sc.recorded_tasks.size();
    f.n_pot_done = sc.potential_tasks.size();
  }
  void idle_filter_init(IdleFilter &f, const Scenario &sc, unsigned int snap_bits) {
    f.k = (int)sc.pending_tasks.size();
    SolverScratch::bump(scr.seen_epoch, scr.seen_stamp);  // no task accounted yet
    for (auto &kv : sweep_topk_idle(f.k, snap_bits)) {
      f.value[kv.second] = kv.first;
      f.sorted.insert(kv.first);
    }
    idle_filter_account(f, sc);
  }
  bool idle_filter_check(IdleFilter &f, const Scenario &sc) {
    idle_filter_account(f, sc);
    if (f.rq.empty() && !sc.pending_tasks.empty()) {  // the pending tasks of a builder never change
      for (int t : sc.pending_tasks) f.rq.push_back(req(t, KAI_RES_GPU));
      std::sort(f.rq.begin(), f.rq.end(), std::greater<double>());
    }
    const std::vector<double> &rq = f.rq;
    if (!rq.empty() && rq[0] != 0 && (f.sorted.empty() || *f.sorted.begin() < rq[0])) return false;  // first requirement unmatched
    std::vector<double> cap;
    for (auto it = f.sorted.begin(); it != f.sorted.end() && (int)cap.size() < f.k; ++it) cap.push_back(*it);
    std::vector<double> used(cap.size(), 0.0);
    for (double required : rq) {
      if (required == 0) return true;
      bool matched = false;
      for (size_t h = 0; h < cap.size(); h++) {
        if (cap[h] < required) break;
        if (cap[h] - used[h] >= required) {
          used[h] += required;
          matched = true;
          break;
        }
      }
      if (!matched) return false;
    }
    return true;
  }

  // ---------------- validators ----------------
  int solver_kind = 0;  // 0 reclaim, 1 consolidation, 2 preempt
  std::vector<double> sim_alloc, sim_np;  // proportion.go:131-136 jobSimulationQueues (allocated columns)
  double SA(int r, int q) const { return sim_alloc[(size_t)r * Q + q]; }
  double SNP(int r, int q) const { return sim_np[(size_t)r * Q + q]; }
  struct Quant {
    double v[QR];
  };
  static bool quant_le(const double *a, const double *b) {
    for (int r = 0; r < QR; r++)
      if (compare_quantities(a[r], b[r]) > 0) return false;
    return true;
  }
  bool can_reclaim_resources(int j) {  // reclaimable.go:29-51
    const double *rq = tta_init_resource(j, false);
    int q = s.j_queue[j];
    for (int r = 0; r < QR; r++)
      if (compare_quantities(QA(r, q) + rq[r], qfair(r, q)) > 0) return false;
    if (preemptible(j)) return true;
    for (int r = 0; r < QR; r++)
      if (compare_quantities(QNP(r, q) + rq[r], qdes(r, q)) > 0) return false;
    return true;
  }
  void leveled_queues(int reclaimer_q, int reclaimee_q, int &a, int &b) const {  // :234-263
    std::vector<int> pa, pb;
    for (int q = reclaimer_q; q >= 0; q = s.q_parent[q]) pa.insert(pa.begin(), q);
    for (int q = reclaimee_q; q >= 0; q = s.q_parent[q]) pb.insert(pb.begin(), q);
    size_t n = std::min(pa.size(), pb.size());
    a = b = -1;
    for (size_t i = 0; i < n; i++) {
      a = pa[i];
      b = pb[i];
      if (a != b) break;
    }
  }
  bool fits_reclaim_strategy(const double *rreq, int reclaimer_q, int reclaimee_q, const double *remaining) const {
    double allocatable[QR], deserved[QR];
    for (int r = 0; r < QR; r++) {
      allocatable[r] = qallocatable(r, reclaimee_q);
      deserved[r] = qdes(r, reclaimee_q);
    }
    if (!quant_le(remaining, allocatable)) return true;  // MaintainFairShareStrategy
    double want[QR], rdes[QR];
    for (int r = 0; r < QR; r++) {
      want[r] = SA(r, reclaimer_q) + rreq[r];
      rdes[r] = qdes(r, reclaimer_q);
    }
    if (!quant_le(want, rdes)) return false;  // GuaranteeDeservedQuotaStrategy
    if (quant_le(remaining, deserved)) return false;
    return true;
  }
  static double saturation_ratio(double allocated, double fair) {
    if (fair == 0) return allocated > 0 ? INFINITY : 0.0;
    if (fair == KAI_UNLIMITED) return 0.0;
    return allocated / fair;
  }
  bool reclaimable(int reclaimer_q, bool reclaimer_preemptible, const double *rreq,
                   const std::map<int, std::vector<Quant>> &by_queue) {  // reclaimable.go:53-220
    std::map<int, Quant> remaining;
    std::map<int, unsigned> involved;
    auto get_remaining = [&](int q) -> Quant & {
      auto it = remaining.find(q);
      if (it == remaining.end()) {
        Quant x;
        for (int r = 0; r < QR; r++) x.v[r] = SA(r, q);
        it = remaining.emplace(q, x).first;
      }
      return it->second;
    };
    for (const auto &kv : by_queue) {
      int leaf = kv.first, lq, eq;
      leveled_queues(reclaimer_q, leaf, lq, eq);
      unsigned m = 0;
      for (const Quant &x : kv.second)
        for (int r = 0; r < QR; r++)
          if (x.v[r] > 0) m |= 1u << r;
      involved[leaf] = m;
      get_remaining(eq);
      for (const Quant &res : kv.second) {
        if (!fits_reclaim_strategy(rreq, lq, eq, get_remaining(eq).v)) return false;
        for (int q = leaf; q >= 0; q = s.q_parent[q]) {
          Quant &rem = get_remaining(q);
          for (int r = 0; r < QR; r++) rem.v[r] -= res.v[r];
          if (involved.count(q))
            involved[q] |= involved[leaf];
          else
            involved[q] = involved[leaf];
        }
      }
    }
    unsigned reclaimer_involved = 0;
    for (int r = 0; r < QR; r++)
      if (rreq[r] > 0) reclaimer_involved |= 1u << r;
    for (int rq = reclaimer_q; rq >= 0; rq = s.q_parent[rq]) {
      Quant mine;
      auto it = remaining.find(rq);
      if (it != remaining.end()) {
        for (int r = 0; r < QR; r++) it->second.v[r] += rreq[r];
        mine = it->second;
      } else {
        for (int r = 0; r < QR; r++) mine.v[r] = SA(r, rq) + rreq[r];
      }
      std::vector<int> sib_ids;
      for (const auto &kv : remaining) sib_ids.push_back(kv.first);
      for (int sib : sib_ids) {
        if (s.q_parent[sib] != s.q_parent[rq] || sib == rq) continue;
        const Quant &sr = remaining[sib];
        unsigned inv = (involved.count(sib) ? involved[sib] : 0u) | reclaimer_involved;
        for (int r = 0; r < QR; r++) {
          if (!(inv & (1u << r))) continue;
          double rf = qfair(r, rq), sf = qfair(r, sib);
          if (rf == KAI_UNLIMITED && sf == KAI_UNLIMITED) continue;
          double ratio_r = saturation_ratio(mine.v[r], rf), ratio_s = saturation_ratio(sr.v[r], sf);
          if (ratio_r > 1 && sf > 0 && ratio_r * cfg.saturation_multiplier >= ratio_s) return false;
        }
      }
      if (reclaimer_preemptible) continue;
      for (int r = 0; r < QR; r++)
        if (compare_quantities(SNP(r, rq) + rreq[r], qdes(r, rq)) > 0) return false;
    }
    return true;
  }
  // ---------------- plugins/minruntime ----------------
  const double *q_preempt_mrt = nullptr, *q_reclaim_mrt = nullptr, *j_last_start = nullptr;  // see kai_engine.h
  const double *j_stale_since = nullptr;                                                      // StalenessInfo.TimeStamp
  double now_s = 0;
  double preempt_min_runtime(int q) const {  // resolver.go:46-67
    for (int c = q; c >= 0; c = s.q_parent[c])
      if (q_preempt_mrt && q_preempt_mrt[c] >= 0) return q_preempt_mrt[c];
    return cfg.default_preempt_min_runtime_s;
  }
  double reclaim_min_runtime(int pq, int vq) const {  // resolver.go:69-187
    if (pq < 0 || vq < 0) return cfg.default_reclaim_min_runtime_s;
    auto set = [&](int q) { return q_reclaim_mrt && q_reclaim_mrt[q] >= 0; };
    if (cfg.reclaim_resolve_method == KAI_RESOLVE_QUEUE) {
      for (int c = vq; c >= 0; c = s.q_parent[c])
        if (set(c)) return q_reclaim_mrt[c];
      return cfg.default_reclaim_min_runtime_s;
    }
    std::vector<int> pp, vp;  // leaf first
    for (int c = pq; c >= 0; c = s.q_parent[c]) pp.push_back(c);
    for (int c = vq; c >= 0; c = s.q_parent[c]) vp.push_back(c);
    const int np = (int)pp.size(), nv = (int)vp.size();
    if (pp[np - 1] != vp[nv - 1])  // different top-level queues: the victim's top-level value
      return set(vp[nv - 1]) ? q_reclaim_mrt[vp[nv - 1]] : cfg.default_reclaim_min_runtime_s;
    int lca = 0;  // depth (root = 0) of the last common queue, then one step down the victim's path if there is one
    for (int i = 0; i < (np < nv ? np : nv); i++) {
      if (pp[np - 1 - i] != vp[nv - 1 - i]) break;
      lca = i;
    }
    if (lca + 1 < nv) lca++;
    for (int i = lca; i >= 0; i--)
      if (set(vp[nv - 1 - i])) return q_reclaim_mrt[vp[nv - 1 - i]];
    return cfg.default_reclaim_min_runtime_s;
  }
  bool job_elastic(int j) const {  // job_info.go:408-415
    for (int ps = ps_begin(j); ps < ps_end(j); ps++)
      if (s.ps_min[ps] < pst_end(ps) - pst_begin(ps)) return true;
    return false;
  }
  bool minruntime_protected(bool reclaim, int pending_job, int victim) const {  // minruntime.go:147-192
    if (!j_last_start || !(j_last_start[victim] > 0)) return false;
    double mrt = reclaim ? reclaim_min_runtime(s.j_queue[pending_job], s.j_queue[victim]) : preempt_min_runtime(s.j_queue[victim]);
    return now_s < j_last_start[victim] + mrt;
  }
  bool minruntime_filter(bool reclaim, int pending_job, int victim) const {  // :93-105
    return job_elastic(victim) || !minruntime_protected(reclaim, pending_job, victim);
  }
  bool minruntime_validator(const Scenario &sc, bool reclaim) const {  // :107-145,206-229
    if (!j_last_start) return true;
    int pj = vjob(sc.preemptor);
    for (const auto &kv : sc.victims) {
      int vj = kv.first;
      if (!job_elastic(vj) || !minruntime_protected(reclaim, pj, vj)) continue;
      for (int ps = ps_begin(vj); ps < ps_end(vj); ps++) {
        int victims = 0;
        for (int t : kv.second)
          if (s.t_podset[t] == ps) victims++;
        if (!victims) continue;
        if (s.ps_min[ps] > count_ps(ps, kActiveUsed) - victims) return false;
      }
    }
    return true;
  }

  bool reclaim_validator(const Scenario &sc) {  // proportion.go:143-240
    int rj = vjob(sc.preemptor);
    const double *rq = tta_init_resource(sc.preemptor, false);
    std::map<int, std::vector<Quant>> by_queue;
    for (const auto &kv : sc.victims) {
      int vj = kv.first;
      std::vector<int> core, elastic;
      for (int ps = ps_begin(vj); ps < ps_end(vj); ps++) {
        int i = 0;
        for (int t : kv.second) {
          if (s.t_podset[t] != ps) continue;
          (i < s.ps_min[ps] ? core : elastic).push_back(t);
          i++;
        }
      }
      auto get_resources = [&](const std::vector<int> &tasks, Quant &out) {
        int n = 0;
        for (int r = 0; r < QR; r++) out.v[r] = 0;
        for (int t : tasks) {
          if (cfg.allow_consolidating_reclaim && (st[t] & kActiveAllocated)) continue;
          n++;
          for (int r = 0; r < QR; r++) out.v[r] += req(t, r);
        }
        return n > 0;
      };
      std::vector<Quant> res;
      for (int t : elastic) {
        Quant x;
        if (get_resources({t}, x)) res.push_back(x);
      }
      Quant x;
      if (get_resources(core, x)) res.push_back(x);
      if (res.empty()) continue;
      auto &dst = by_queue[s.j_queue[vj]];
      dst.insert(dst.end(), res.begin(), res.end());
    }
    return reclaimable(s.j_queue[rj], preemptible(rj), rq, by_queue);
  }
  bool consolidation_validator(const Scenario &sc) const {  // consolidation.go:108-117
    for (const auto &kv : sc.victims)
      for (int t : kv.second)
        if (st[t] == KAI_POD_RELEASING) return false;
    return true;
  }

  // ---------------- simulation (actions/common/action.go:67-122) ----------------
  JobsOrder sim_order;  // the job order of the current simulation (kept for its capacity)
  bool try_virtually_allocate(const Scenario &sc, const std::vector<int> &victim_tasks) {
    const int pj = vjob(sc.preemptor);
    simulations++;
    const double t_setup0 = HostBackend::now();
    std::set<int> in_set(pending_jobs), victim_jobs;
    for (int t : victim_tasks) {
      in_set.insert(tjob(t));
      victim_jobs.insert(tjob(t));
    }
    in_set.insert(pj);
    std::vector<int> vs;
    for (int j : in_set) vs.push_back(j == pj ? sc.preemptor : j);  // ascending job index, as before
    JobsOrder &jo = sim_order;
    jo.init(this, false);
    init_jobs_order(jo, vs, OrderOpts());
    t_sim_setup += HostBackend::now() - t_setup0;
    bool preemptor_allocated = false;
    while (!jo.is_empty() && !gpu_failed()) {
      int v = jo.pop_next_job();
      if (v < 0) break;
      int j = vjob(v);
      if (j != pj && !victim_jobs.count(j)) continue;
      tta_init_resource(v, false);
      if (j != pj) {
        allocate_job(v);
        continue;
      }
      if (!allocate_job(v)) return false;
      preemptor_allocated = true;
    }
    return preemptor_allocated;
  }

  struct SolveResult {
    bool has = false, solved = false;
    std::vector<int> victim_tasks, victim_jobs;
  };
  SolveResult run_simulation(Scenario &sc, const std::vector<int> &victim_tasks) {  // by_pod_solver.go:124-143,229-253
    SolveResult res;
    if (!try_virtually_allocate(sc, victim_tasks)) return res;
    std::vector<int> preempted, pipelined;
    for (int t : victim_tasks) {
      if (st[t] == KAI_POD_RELEASING)
        preempted.push_back(t);
      else if (st[t] == KAI_POD_PIPELINED)
        pipelined.push_back(t);
    }
    res.has = true;
    // every registered validator must accept (session_plugins.go:135-164): reclaim = proportion + minruntime,
    // preempt = minruntime, consolidation = its own closure
    bool valid = solver_kind == 0 ? (reclaim_validator(sc) && minruntime_validator(sc, true))
                                  : (solver_kind == 1 ? consolidation_validator(sc) : minruntime_validator(sc, false));
    if (!valid) {
      stmt_discard();
      return res;
    }
    res.victim_tasks = preempted;
    res.victim_tasks.insert(res.victim_tasks.end(), pipelined.begin(), pipelined.end());
    std::map<int, std::vector<int>> groups;  // getVictimJobsFromVictimTasks
    for (int t : res.victim_tasks) {
      int j = tjob(t);
      bool exists = false;
      for (int g : groups[j]) {
        std::vector<int> gt = v_all_tasks(g);
        if (std::find(gt.begin(), gt.end(), t) != gt.end()) exists = true;
      }
      if (exists) continue;
      for (int g : sc.task_groups[j]) {
        std::vector<int> gt = v_all_tasks(g);
        if (std::find(gt.begin(), gt.end(), t) != gt.end()) {
          groups[j].push_back(g);
          break;
        }
      }
    }
    for (auto &kv : groups) res.victim_jobs.insert(res.victim_jobs.end(), kv.second.begin(), kv.second.end());
    res.solved = true;
    return res;
  }

  // feasible-node set: host knows membership (base from the attempt-start state + extras), the scanners hold the bits
  bool feas_all = false;
  std::vector<char> feas_extra;      // per node: added beyond the base set
  std::vector<int> feas_extra_list;  // nodes currently flagged on the GPU beyond the base set
  bool in_base(int n) const { return feas_all || start_Ig(n) > 0 || start_Lg(n) > 0; }
  bool feas_add(int n) {  // true if the node was not in the set
    if (in_base(n) || feas_extra[n]) return false;
    feas_extra[n] = 1;
    feas_extra_list.push_back(n);
    emit_delta(seq, n, ND_FEAS_SET, 0);
    return true;
  }
  void feas_remove(int n) {
    if (!feas_extra[n]) return;
    feas_extra[n] = 0;
    feas_extra_list.erase(std::find(feas_extra_list.begin(), feas_extra_list.end(), n));
    emit_delta(seq, n, ND_FEAS_CLR, 0);
  }
  void feas_clear_extras() {
    std::vector<int> l = feas_extra_list;
    for (int n : l) feas_remove(n);
  }

  SolveResult bypod_solve(Scenario &sc) {  // by_pod_solver.go:69-122,145-201
    ops_truncate(0);
    {
      const double t0 = HostBackend::now();
      for (int t : sc.recorded_tasks) stmt_evict(t);
      t_evict += HostBackend::now() - t0;
    }
    if (sc.potential_tasks.empty()) {
      if (!sc.recorded_tasks.empty()) {
        SolveResult r = run_simulation(sc, sc.recorded_tasks);
        if (r.has) return r;
      }
    } else {
      int latest = tjob(sc.potential_tasks.back());
      std::vector<int> nodes;
      for (int ps = ps_begin(latest); ps < ps_end(latest); ps++)
        for (int t = pst_begin(ps); t < pst_end(ps); t++)
          if (tn[t] >= 0 && std::find(nodes.begin(), nodes.end(), tn[t]) == nodes.end()) nodes.push_back(tn[t]);
      std::sort(nodes.begin(), nodes.end());
      for (int node : nodes) {
        if (gpu_failed()) break;
        int cp = stmt_checkpoint();
        std::vector<int> potential = scenario_victims_from_node(sc, node);
        for (int t : potential) stmt_evict(t);
        std::vector<int> added;
        for (int t : potential)
          if (feas_add(tn[t])) added.push_back(tn[t]);
        std::vector<int> victim_tasks = sc.recorded_tasks;
        victim_tasks.insert(victim_tasks.end(), potential.begin(), potential.end());
        SolveResult r = run_simulation(sc, victim_tasks);
        if (r.has) return r;
        for (int n : added) feas_remove(n);
        stmt_rollback(cp);
      }
    }
    stmt_discard();
    SolveResult none;
    none.has = true;
    return none;
  }

  // Victims-queue cache.  The reference rebuilds the victims JobsOrderByQueues for every partial job of every
  // reclaimer from ALL jobs of the session (reclaim.go:121-143, consolidation.go:119-157) — O(jobs) heap pushes each
  // time.  Here the eligible victims of a leaf queue are kept in pop order (inverse JobOrderFn = descending packed
  // key: priority, elastic class, creation / UID rank) and rebuilt only when a task of that queue changed status
  // since (leaf_epoch).  A sorted run pushed in order IS the heap those pushes build (no sift moves anything), and a
  // leaf is linked into its ancestors' heaps with its best job on top either way, so the tree below is the one
  // push_job would have produced, queue by queue in ascending order.
  std::vector<std::vector<int>> vq_leaf;
  std::vector<long long> vq_leaf_epoch, leaf_epoch, vq_top_epoch;
  std::vector<int> vq_top;  // best victim of the leaf (-1: none), valid while vq_top_epoch matches
  long long vq_rebuilt = 0, vq_reused = 0;
  unsigned long long victim_key(JobsOrder &jo, int j) {
    bool below, above, exactly;
    jo.min_available_state(j, below, above, exactly);
    return make_job_key(s.j_priority[j], below ? 0 : (exactly ? 1 : 2), s.j_order_rank[j]);
  }
  int victim_leaf_top(JobsOrder &jo, int q) {
    if (vq_top_epoch[q] == leaf_epoch[q]) return vq_top[q];
    const double tt = HostBackend::now();
    int best = -1;
    unsigned long long best_key = 0;
    for (int i = s.q_job_begin[q]; i < s.q_job_begin[q + 1]; i++) {
      const int j = s.q_jobs_sorted[i];
      if (!preemptible(j) || count_job(j, kActiveAllocated) == 0) continue;
      const unsigned long long k = victim_key(jo, j);
      if (best < 0 || k > best_key) {
        best = j;
        best_key = k;
      }
    }
    vq_top[q] = best;
    vq_top_epoch[q] = leaf_epoch[q];
    t_vq_top += HostBackend::now() - tt;
    return best;
  }
  const std::vector<int> &victim_leaf_list(JobsOrder &jo, int q) {
    if (vq_leaf_epoch[q] == leaf_epoch[q]) {
      vq_reused++;
      return vq_leaf[q];
    }
    vq_rebuilt++;
    std::vector<std::pair<unsigned long long, int>> keyed;
    for (int i = s.q_job_begin[q]; i < s.q_job_begin[q + 1]; i++) {
      const int j = s.q_jobs_sorted[i];
      if (!preemptible(j) || count_job(j, kActiveAllocated) == 0) continue;
      keyed.push_back({victim_key(jo, j), j});
    }
    std::sort(keyed.begin(), keyed.end(), [](const std::pair<unsigned long long, int> &a, const std::pair<unsigned long long, int> &b) { return a.first > b.first; });
    vq_leaf[q].clear();
    for (auto &kv : keyed) vq_leaf[q].push_back(kv.second);
    vq_leaf_epoch[q] = leaf_epoch[q];
    return vq_leaf[q];
  }
  bool build_victims_queue_cached(JobsOrder &jo, int pending_job) {
    if (solver_kind == 2 || j_last_start || getenv("KAI_NO_VICTIM_CACHE")) return false;  // preempt: one queue; min-runtime filters depend on the pair
    if (solver_kind == 1 && cfg.max_consolidation_preemptees != -1) return false;
    if (!ops.empty()) return false;  // built on the committed state only
    const int pq = s.j_queue[pending_job];
    for (int q = 0; q < Q; q++) {
      if (s.q_nchildren[q] != 0 || s.q_job_begin[q + 1] == s.q_job_begin[q]) continue;
      if (solver_kind == 0 && q == pq) continue;  // reclaim.go:126: other queues only
      if (solver_kind == 1 && q == pq) {  // consolidation.go:127: every job of the queue but the pending one
        std::vector<int> a = victim_leaf_list(jo, q);
        a.erase(std::remove(a.begin(), a.end(), pending_job), a.end());
        if (a.empty()) continue;
        const int leaf = jo.make_node(q, true);
        jo.queue_node[q] = leaf;
        jo.heap_assign(leaf, a.data(), (int)a.size());
        jo.ensure_chain(leaf);
        jo.mark_ancestors(leaf);
        continue;
      }
      // only the leaf's best job is needed until the leaf itself is popped: the rest of its run is loaded then
      const int top = victim_leaf_top(jo, q);
      if (top < 0) continue;
      const int leaf = jo.make_node(q, true);
      jo.queue_node[q] = leaf;
      jo.heap_assign(leaf, &top, 1);
      jo.nodes[leaf].lazy_queue = q;
      jo.ensure_chain(leaf);
      jo.mark_ancestors(leaf);
    }
    return true;
  }
  // the partial jobs of one pending job (job_solver.go:60-88) start from the same committed state: the queue built for
  // the first one is copied for the others (commit_epoch counts the statements committed in this action)
  JobsOrder vq_proto, vq_cur;  // vq_cur: the victims queue of the partial job being solved (kept for its capacity)
  int vq_proto_job = -1, vq_proto_kind = -1;
  long long vq_proto_commit = -1, commit_epoch = 0;
  void build_victims_queue(JobsOrder &jo, int pending_job) {
    if (vq_proto_job == pending_job && vq_proto_kind == solver_kind && vq_proto_commit == commit_epoch && ops.empty() &&
        !getenv("KAI_NO_VICTIM_CACHE")) {
      const double tc = HostBackend::now();
      jo.copy_from(vq_proto);
      t_vq_copy += HostBackend::now() - tc;
      n_vq_copy++;
      return;
    }
    n_vq_build++;
    jo.init(this, true);
    if (build_victims_queue_cached(jo, pending_job)) {
      vq_proto.copy_from(jo);
      vq_proto_job = pending_job;
      vq_proto_kind = solver_kind;
      vq_proto_commit = commit_epoch;
      return;
    }
    std::vector<int> vs;
    OrderOpts op;
    if (solver_kind == 0) {  // reclaim.go:121-143
      op.filter_non_preemptible = true;
      op.filter_non_active_allocated = true;
      for (int j = 0; j < J; j++)
        if (s.j_queue[j] != s.j_queue[pending_job] && minruntime_filter(true, pending_job, j)) vs.push_back(j);
    } else if (solver_kind == 2) {  // preempt.go:125-161 + utils/action.go:20-52
      for (int j = 0; j < J; j++) {
        if (count_job(j, kAlive) == 0) continue;
        if (!preemptible(j) || s.j_priority[j] >= s.j_priority[pending_job]) continue;
        if (s.j_queue[j] != s.j_queue[pending_job] || j == pending_job) continue;
        if (count_job(j, kActiveAllocated) == 0) continue;
        if (!minruntime_filter(false, pending_job, j)) continue;
        vs.push_back(j);
      }
    } else {  // consolidation.go:119-157 + utils/action.go:20-52
      int counter = 0;
      for (int j = 0; j < J; j++) {
        if (count_job(j, kAlive) == 0) continue;
        if (!preemptible(j) || j == pending_job) continue;
        if (cfg.max_consolidation_preemptees != -1 && counter > cfg.max_consolidation_preemptees) continue;
        if (count_job(j, kActiveAllocated) == 0) continue;
        counter++;
        vs.push_back(j);
      }
    }
    init_jobs_order(jo, vs, op);
  }

  struct SolveState {
    std::vector<int> recorded_jobs, recorded_tasks;
  };
  unsigned int pending_snap_bits = 0;  // feasible-set snapshot still to be attached to the next TOPK record
  SolveResult solve_partial(const SolveState &state, int pending_job, int partial) {  // job_solver.go:90-118
    feas_clear_extras();
    for (int t : state.recorded_tasks)
      if (tn[t] >= 0) feas_add(tn[t]);
    Scenario sc;
    sc.preemptor = partial;
    sc.pending_tasks = v_all_tasks(partial);
    sc.recorded_jobs = state.recorded_jobs;
    for (int rv : state.recorded_jobs) scenario_append_group(sc, v_all_tasks(rv));
    for (int rv : state.recorded_jobs)
      for (int t : v_all_tasks(rv)) sc.recorded_tasks.push_back(t);
    const unsigned rec = SolverScratch::bump(scr.rec_epoch, scr.rec_stamp);
    for (int t : sc.recorded_tasks) scr.rec_stamp[t] = rec;
    JobsOrder &victims_queue = vq_cur;
    {
      const double t0 = HostBackend::now();
      build_victims_queue(victims_queue, pending_job);
      t_victims_queue += HostBackend::now() - t0;
    }
    IdleFilter filter;
    const double tfi = HostBackend::now();
    idle_filter_init(filter, sc, pending_snap_bits);
    t_finit += HostBackend::now() - tfi;
    pending_snap_bits = 0;
    bool first = true;
    while (!gpu_failed()) {
      bool need_add = !first, have = false;
      first = false;
      for (;;) {
        if (need_add) {
          bool added = false;
          while (!added) {
            if (victims_queue.is_empty()) break;
            double tq = HostBackend::now();
            int next = victims_queue.pop_next_job();
            t_vq_pop += HostBackend::now() - tq;
            if (next < 0) break;
            bool has_more = false;
            tq = HostBackend::now();
            std::vector<int> tasks = tasks_to_evict(next, has_more);
            t_tte += HostBackend::now() - tq;
            bool hit = false;
            for (int t : tasks)
              if (scr.rec_stamp[t] == rec) hit = true;
            if (hit) {
              std::vector<int> remaining;
              for (int t : v_all_tasks(next))
                if (scr.rec_stamp[t] != rec) remaining.push_back(t);
              if (!remaining.empty()) victims_queue.push_job(make_clone(next, remaining));
              continue;
            }
            if (has_more) {
              std::vector<int> remaining;
              for (int t : v_all_tasks(next))
                if (std::find(tasks.begin(), tasks.end(), t) == tasks.end()) remaining.push_back(t);
              victims_queue.push_job(make_clone(next, remaining));
            }
            tq = HostBackend::now();
            scenario_add_potential(sc, tasks);
            t_addp += HostBackend::now() - tq;
            added = true;
          }
          if (!added) break;
        }
        const double tf = HostBackend::now();
        const bool fc = idle_filter_check(filter, sc);
        t_filter += HostBackend::now() - tf;
        if (fc) {
          have = true;
          break;
        }
        need_add = true;
      }
      if (!have) break;
      scenarios++;
      const double tb = HostBackend::now();
      SolveResult r = bypod_solve(sc);
      t_bypod += HostBackend::now() - tb;
      if (r.solved) return r;
    }
    return SolveResult();
  }

  bool solve_job(int j) {  // job_solver.go:47-88,120-148
    SolveState state;
    int original_active = count_job(j, kActiveUsed);
    std::vector<int> tta = tasks_to_allocate(j, false);
    std::vector<int> pending;
    bool have_statement = false;
    for (size_t i = 0; i < tta.size() && !gpu_failed(); i++) {
      pending.push_back(tta[i]);
      bool satisfactory = pending.size() == tta.size();
      int partial = make_clone(j, pending);
      {
        View &pv = views[partial - J];
        for (size_t k = 0; k < pv.ps_tasks.size(); k++)
          if (!pv.ps_tasks[k].empty()) pv.ps_min[k] = (int)pv.ps_tasks[k].size();
      }
      SolveResult r = solve_partial(state, j, partial);
      if (!r.solved) {
        have_statement = false;
        break;
      }
      if (!satisfactory) stmt_discard();
      have_statement = satisfactory;
      state.recorded_tasks = r.victim_tasks;
      state.recorded_jobs = r.victim_jobs;
    }
    int active = count_job(j, kActiveUsed);
    bool solved = true;
    for (int ps = ps_begin(j); ps < ps_end(j); ps++)
      if (count_ps(ps, kActiveUsed) < s.ps_min[ps]) solved = false;
    if (original_active >= active) solved = false;
    if (!have_statement) ops_truncate(0);
    return solved;
  }
  // starts a job attempt: the next TOPK record snapshots FeasibleNodesForJob (feasible_nodes.go:11-26)
  void begin_attempt(int j) {
    SolverScratch::bump(scr.node_epoch, scr.node_stamp);
    for (int n : feas_extra_list) feas_extra[n] = 0;  // feas_extra is set exactly on feas_extra_list
    feas_extra_list.clear();
    feas_all = false;
    for (int ps = ps_begin(j); ps < ps_end(j); ps++)
      for (int t = pst_begin(ps); t < pst_end(ps); t++)
        if (!(req(t, KAI_RES_GPU) > 0)) feas_all = true;
    pending_snap_bits = feas_all ? XB_SNAP_ALL : XB_SNAP_GPUFREE;
    views.clear();
    // No node changes before that TOPK record, so the rows it will flag are the GPU-free rows of now (= in_base()).
    base_known = host_sweep_max > 0 && !feas_all && gpu_free_list.size() <= (size_t)host_sweep_max;
    if (base_known) base_list = gpu_free_list;
  }

  // ---------------- minimal_job_comparison.go ----------------
  bool req_le(int a, int b) const {
    for (int r = 0; r < R; r++) {
      if (r >= 3) {
        if (req(a, r) != 0 && req(a, r) > req(b, r)) return false;
      } else if (req(a, r) > req(b, r))
        return false;
    }
    return true;
  }
  std::vector<int> sorted_pending(int j) const {
    std::vector<int> v;
    for (int ps = ps_begin(j); ps < ps_end(j); ps++)
      for (int t = pst_begin(ps); t < pst_end(ps); t++)
        if (st[t] == KAI_POD_PENDING) v.push_back(t);
    for (size_t i = 1; i < v.size(); i++)
      for (size_t k = i; k > 0 && req_le(v[k], v[k - 1]); k--) std::swap(v[k], v[k - 1]);
    return v;
  }
  typedef std::map<int, int> Reps;
  bool easier_to_schedule(const Reps &m, int j) const {
    if (!job_signature || job_signature[j] < 0) return true;
    auto it = m.find(job_signature[j]);
    if (it == m.end()) return true;
    std::vector<int> a = sorted_pending(j), b = sorted_pending(it->second);
    if (a.empty() || b.empty()) return false;
    if (b.size() > a.size()) return true;
    for (size_t i = 0; i < a.size(); i++) {
      if (i >= b.size()) return false;
      if (req_le(a[i], b[i])) {
        if (req_le(b[i], a[i])) continue;
        return true;
      }
    }
    return false;
  }
  void update_representative(Reps &m, int j) const {
    if (!job_signature || job_signature[j] < 0) return;
    auto it = m.find(job_signature[j]);
    if (it != m.end()) {
      std::vector<int> a = sorted_pending(j), b = sorted_pending(it->second);
      bool smaller = !(a.empty() || b.empty()) && a.size() <= b.size();
      if (smaller)
        for (size_t i = 0; i < a.size(); i++)
          if (!req_le(a[i], b[i])) smaller = false;
      if (!smaller) return;
    }
    m[job_signature[j]] = j;
  }

  // KAI_SOLVER_SETUP_CHECK (tests): recount what prepare() took from the prepare kernels by scanning every task status,
  // and fail the action on any difference
  bool setup_check = false;
  void setup_fail(const char *field, int index, long long got, long long want) {
    snprintf(hb.error_msg, sizeof(hb.error_msg), "KAI_SOLVER_SETUP_CHECK: %s[%d] is %lld, a recount of the task statuses gives %lld",
             field, index, got, want);
    seq.error = kSeqErrHostSweep;
  }
  void check_setup_counts() {
    std::vector<int> act(S, 0), pend(J, 0);
    for (int t = 0; t < T; t++) {
      if (st[t] == KAI_POD_PENDING) pend[tjob(t)]++;
      if (st[t] & kActiveAllocated) act[s.t_podset[t]]++;
    }
    for (int ps = 0; ps < S; ps++)
      if (ps_active[ps] != act[ps]) return setup_fail("ps_active", ps, ps_active[ps], act[ps]);
    for (int j = 0; j < J; j++) {
      if (pending_cnt[j] != pend[j]) return setup_fail("pending_cnt", j, pending_cnt[j], pend[j]);
      if ((pending_jobs.count(j) != 0) != (pend[j] > 0)) return setup_fail("pending_jobs", j, (long long)pending_jobs.count(j), pend[j] > 0);
    }
  }

  double t_prepare = 0;
  void prepare() {
    const double t0 = HostBackend::now();
    SolverScratch::bump(scr.job_epoch, scr.job_cache, &Cache::stamp);  // every job cache of an earlier action is stale
    SolverScratch::bump(scr.node_epoch, scr.node_stamp);
    vq_leaf.assign(Q, {});
    vq_leaf_epoch.assign(Q, -1);
    vq_top.assign(Q, -1);
    vq_top_epoch.assign(Q, -1);
    leaf_epoch.assign(Q, 0);
    // per-podset active-allocated and pending counts from k_prep_jobs (ps_cnt0, same masks, over the statuses this
    // action starts from: nothing changes a status between that kernel's copy-back and here)
    ps_active.assign(s.ps_cnt0, s.ps_cnt0 + S);
    pending_cnt.assign(J, 0);
    pending_jobs.clear();
    for (int j = 0; j < J; j++) {
      int c = 0;
      for (int ps = ps_begin(j); ps < ps_end(j); ps++) c += s.ps_cnt0[S + ps];
      pending_cnt[j] = c;
      if (c > 0) pending_jobs.insert(pending_jobs.end(), j);
    }
    if (setup_check) check_setup_counts();
    feas_extra.assign(N, 0);
    feas_extra_list.clear();
    ops_truncate(0);
    free_ready = 0;  // once per action, from the mirror of the GPU column the action starts with
    base_known = false;
    gpu_free_list.clear();
    if (host_sweep_max > 0) gpu_free_pos.assign(N, -1);
    for (int n = 0; n < N; n++) {
      if (s.nflags[n] & KAI_NODE_READY) free_ready += Ig(n) + Lg(n);
      if (host_sweep_max > 0) gpu_free_update(n);
    }
    t_prepare += HostBackend::now() - t0;
  }

  // ---------------- actions/reclaim/reclaim.go:46-119 ----------------
  void run_reclaim() {
    solver_kind = 0;
    prepare();
    JobsOrder jo;
    jo.init(this, false);
    {
      std::vector<int> vs(pending_jobs.begin(), pending_jobs.end());  // filter_non_pending: jobs with Pending tasks only
      OrderOpts op;
      op.filter_non_pending = op.filter_unready = true;
      init_jobs_order(jo, vs, op);
    }
    std::map<int, Reps> failed_by_queue;
    while (!jo.is_empty() && !gpu_failed()) {
      int j = jo.pop_next_job();
      if (j < 0) break;
      if (!can_reclaim_resources(j)) continue;
      Reps &reps = failed_by_queue[s.j_queue[j]];
      if (use_signatures && !easier_to_schedule(reps, j)) continue;
      tta_init_resource(j, false);
      sim_alloc.assign(qa, qa + (size_t)QR * Q);  // OnJobSolutionStart
      sim_np.assign(qnp, qnp + (size_t)QR * Q);
      begin_attempt(j);
      bool ok = solve_job(j);
      if (ok) {
        stmt_commit();
        record_visit(seq, j, 1);
      } else {
        ops_truncate(0);
        update_representative(reps, j);
        record_visit(seq, j, 0);
      }
    }
  }
  // ---------------- actions/stalegangeviction/stalegangeviction.go:29-95 ----------------
  void run_stale_gang_eviction() {
    prepare();
    if (cfg.staleness_grace_period_s < 0) return;  // :47-50 negative duration means no eviction
    for (int j = 0; j < J && !gpu_failed(); j++) {
      // :42-57 nil TimeStamp = stamped now = zero time in stale state; else time.Since(TimeStamp) at the snapshot's instant
      double in_stale = (j_stale_since && j_stale_since[j] > 0) ? now_s - j_stale_since[j] : 0.0;
      if (in_stale < double(cfg.staleness_grace_period_s)) continue;
      if (count_job(j, KAI_POD_SUCCEEDED) > 0 || count_job(j, kActiveUsed) == 0) continue;  // job_info.go:417-432
      bool stale = false;
      for (int ps = ps_begin(j); ps < ps_end(j); ps++)
        if (count_ps(ps, kActiveUsed) < s.ps_min[ps]) stale = true;
      if (!stale) continue;
      for (int ps = ps_begin(j); ps < ps_end(j); ps++)
        for (int t = pst_begin(ps); t < pst_end(ps); t++) {
          if (!(st[t] & kActiveAllocated)) continue;
          set_status(t, KAI_POD_RELEASING);  // framework/session.go:127-150 Session.Evict
          node_remove_task(t, tn[t]);
          node_add_task(t);
          queue_allocate(t, false);
          seq.pods_evicted++;
        }
      record_visit(seq, j, 1);
    }
  }
  // ---------------- actions/preempt/preempt.go:46-123 ----------------
  void run_preempt() {
    solver_kind = 2;
    prepare();
    JobsOrder jo;
    jo.init(this, false);
    {
      std::vector<int> vs(pending_jobs.begin(), pending_jobs.end());  // filter_non_pending: jobs with Pending tasks only
      OrderOpts op;
      op.filter_non_pending = op.filter_unready = true;
      init_jobs_order(jo, vs, op);
    }
    std::map<int, Reps> failed_by_queue;
    while (!jo.is_empty() && !gpu_failed()) {
      int j = jo.pop_next_job();
      if (j < 0) break;
      Reps &reps = failed_by_queue[s.j_queue[j]];
      if (use_signatures && !easier_to_schedule(reps, j)) continue;
      tta_init_resource(j, false);
      double rq[QR] = {0, 0, 0};
      for (int t : tasks_to_allocate(j, false))
        for (int r = 0; r < QR; r++) rq[r] += req(t, r);
      bool over_quota = false;  // IsNonPreemptibleJobOverQueueQuotaFn (capacity_policy.go:38-49)
      if (!preemptible(j))
        for (int q = s.j_queue[j]; q >= 0 && !over_quota; q = s.q_parent[q])
          for (int r = 0; r < QR; r++) {
            if (qdes(r, q) == KAI_UNLIMITED || rq[r] == 0) continue;
            if (qdes(r, q) < QNP(r, q) + rq[r]) over_quota = true;
          }
      bool ok = false;
      ops_truncate(0);
      if (!over_quota) {
        begin_attempt(j);
        ok = solve_job(j);
      }
      if (ok) {
        stmt_commit();
        record_visit(seq, j, 1);
      } else {
        ops_truncate(0);
        update_representative(reps, j);
        record_visit(seq, j, 0);
      }
    }
  }
  // ---------------- actions/consolidation/consolidation.go:32-106 ----------------
  void run_consolidation() {
    solver_kind = 1;
    prepare();
    if (cfg.max_consolidation_preemptees == 0) return;
    JobsOrder jo;
    jo.init(this, false);
    {
      std::vector<int> vs(pending_jobs.begin(), pending_jobs.end());
      OrderOpts op;
      op.filter_non_pending = op.filter_unready = op.filter_non_preemptible = true;
      init_jobs_order(jo, vs, op);
    }
    Reps reps;
    while (!jo.is_empty() && !gpu_failed()) {
      int j = jo.pop_next_job();
      if (j < 0) break;
      if (use_signatures && !easier_to_schedule(reps, j)) continue;
      tta_init_resource(j, false);
      // utils/action.go:130-160 IsEnoughGPUsAllocatableForJob: Σ idle + releasing GPUs of ready nodes
      double sum = free_ready, want = 0;
      for (int t : tasks_to_allocate(j, false)) want += req(t, KAI_RES_GPU);
      bool ok = false;
      ops_truncate(0);
      if (sum >= want) {
        begin_attempt(j);
        ok = solve_job(j);
      }
      if (ok) {
        stmt_commit();
        record_visit(seq, j, 1);
      } else {
        ops_truncate(0);
        update_representative(reps, j);
        record_visit(seq, j, 0);
      }
    }
  }
};

}  // namespace kai
