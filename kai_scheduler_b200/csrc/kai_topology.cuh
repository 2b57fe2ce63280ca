// kai_topology.cuh — host side of the topology plugin (row a18) for the host-sequenced engine.
//
// Replaces: plugins/topology/topology_plugin.go:57-110 (domain tree from node labels), job_filtering.go:34-527
// (subSetNodesFn: lowest common domain, per-domain free resources and allocatable pods, bin-packing order of the
// tree, candidate domains bottom-up) and node_scoring.go:36-68 (preferred-level node scores).  Scope: the topology
// constraint of the job's root SubGroupSet.
//
// Division of work: the host keeps the domain trees and evaluates them against its mirror of the node tables (which
// follows every node delta); the GPU does what is per (pod, node): the scanners carry one domain id per level and
// row, an EXT_SELECT entry turns a domain into the row set of the following sweeps (XB_RESTRICT_DOM), and the
// preferred-level score of a row is a table look-up by its domain id (EXT_SCORE entries), added as the last
// NodeOrderFn term.  Children of a domain that sortTree never reaches keep ascending DomainID order (the reference:
// node map iteration order).  Host-only code.
#pragma once
#include <algorithm>
#include <cmath>
#include <array>
#include <functional>
#include <map>
#include <vector>

#include "kai_seq.cuh"

namespace kai {

struct TopologyHost {
  struct Dom {
    int level = -1;  // global level index, -1 = root
    int id = 0;      // dense id inside the level (ascending DomainID order)
    int parent = -1;
    std::vector<int> children, nodes;
    int alloc_pods = -1;  // allocatablePodsNotSet
    double free[KAI_MAX_RES] = {0};
    double free_live[KAI_MAX_RES] = {0};  // Σ Idle + Releasing of the domain's nodes, kept incrementally (all levels)
  };
  struct Topo {
    int lb = 0, le = 0;
    std::vector<Dom> doms;                 // doms[0] = root
    std::vector<std::vector<int>> dom_at;  // [level - lb][id] -> index into doms
    std::vector<char> node_in;
    std::vector<char> lcd_all;  // per level: do all topology nodes share one domain (lowest common domain of the full set)
  };
  int N = 0, R = 4;
  std::vector<int> level_begin, node_domain;
  // SubGroupSet tree, normalised at load (every job has a root set); constraints = (topology, required, preferred)
  std::vector<int> set_parent, set_rank, job_root_set, ps_set;
  std::vector<std::vector<int>> set_children, set_podsets;
  std::vector<std::array<int, 3>> set_con, ps_con;
  std::vector<char> job_general;  // nested sets or any topology constraint: the allocation walks the tree
  const int *t_podset = nullptr;  // [T] (engine task numbering)
  std::vector<Topo> topos;
  const double *mirror = nullptr;  // host mirror of Idle / Releasing, node-major [N][2][R]
  double mI_(int r, int n) const { return mirror[(size_t)n * 2 * R + r]; }
  double mL_(int r, int n) const { return mirror[(size_t)n * 2 * R + R + r]; }
  const double *t_req = nullptr;              // [T][R] (engine task numbering)

  // ---- incremental state, fed by the node-delta stream (Seq::on_node_changed) ----
  // The reference recomputes, per constrained job, the free resources of every domain of the subtree and, per node,
  // how many copies of the job's largest pod fit.  Here the per-leaf-domain sums and, per pod shape ("class"), the
  // per-node counts and their per-leaf-domain sums are kept up to date as nodes change, so that a job costs
  // O(domains), not O(nodes).  (Sums of integer-valued quantities: the order of accumulation is immaterial.)
  bool live = false;
  std::vector<std::vector<int>> leaf_of;  // [topology][node] -> lowest-level domain (index into doms) or -1
  struct PodClass {
    int topo = -1;
    std::vector<double> max_pod;
    bool only_pods = false;
    std::vector<int> cnt;       // [N] calcNodeAccommodation of the node
    std::vector<int> leaf_cnt;  // [doms] sum over the nodes of the domain (every level)
    unsigned long long stamp = 0;
  };
  std::vector<PodClass> classes;
  unsigned long long class_clock = 0;

  int ND(int level, int n) const { return node_domain[(size_t)level * N + n]; }
  // job_filtering.go:213-247 calcNodeAccommodation: the k-th test pod is k copies of the largest pod, accumulated
  int count_node(const std::vector<double> &max_pod, int n) const {
    double acc[KAI_MAX_RES] = {0};
    int cnt = 0;
    for (;;) {
      for (int r = 0; r < R; r++) acc[r] += max_pod[r];
      for (int r = 0; r < R; r++) {
        double a = avail(r, n);
        if (r >= 3) {
          if (acc[r] != 0 && acc[r] > a) return cnt;
        } else if (acc[r] > a)
          return cnt;
      }
      cnt++;
    }
  }
  void ensure_live() {
    if (live) return;
    leaf_of.assign(topos.size(), {});
    for (size_t k = 0; k < topos.size(); k++) {
      Topo &tp = topos[k];
      leaf_of[k].assign(N, -1);
      for (size_t di = 0; di < tp.doms.size(); di++) {
        Dom &d = tp.doms[di];
        for (int r = 0; r < KAI_MAX_RES; r++) d.free_live[r] = 0;
        if (!d.children.empty() || d.level < 0) continue;
        for (int n : d.nodes) {
          leaf_of[k][n] = (int)di;
          for (int r = 0; r < R; r++) {
            d.free_live[r] += mI_(r, n);
            d.free_live[r] += mL_(r, n);
          }
        }
      }
    }
    for (size_t k = 0; k < topos.size(); k++) {  // aggregate upwards: children have larger indices than parents
      Topo &tp = topos[k];
      for (size_t di = tp.doms.size(); di-- > 1;)
        for (int r = 0; r < R; r++) tp.doms[tp.doms[di].parent].free_live[r] += tp.doms[di].free_live[r];
    }
    classes.clear();
    ratio_classes.clear();
    cur_ratio = nullptr;
    dom_ver.assign(topos.size(), {});
    for (size_t k = 0; k < topos.size(); k++) dom_ver[k].assign(topos[k].doms.size(), 1u);
    live = true;
  }
  static void node_changed_hook(void *self, int node, const double *before, const double *after) {
    ((TopologyHost *)self)->node_changed(node, before, after);
  }
  void node_changed(int node, const double *before, const double *after) {
    if (!live) return;
    for (size_t k = 0; k < topos.size(); k++) {
      int leaf = leaf_of[k][node];
      if (leaf < 0) continue;
      for (int d = leaf; d >= 0; d = topos[k].doms[d].parent) {
        for (int r = 0; r < R; r++) topos[k].doms[d].free_live[r] += after[r] - before[r];
        dom_ver[k][d]++;
      }
    }
    for (PodClass &c : classes) {
      int leaf = leaf_of[c.topo][node];
      if (leaf < 0 || c.only_pods) continue;
      int nc = count_node(c.max_pod, node);
      if (nc != c.cnt[node])
        for (int d = leaf; d >= 0; d = topos[c.topo].doms[d].parent) c.leaf_cnt[d] += nc - c.cnt[node];
      c.cnt[node] = nc;
    }
  }
  PodClass &pod_class(int k, const std::vector<double> &max_pod) {
    for (PodClass &c : classes)
      if (c.topo == k && c.max_pod == max_pod) {
        c.stamp = ++class_clock;
        return c;
      }
    if (classes.size() >= 4) {  // evict the least recently used shape
      size_t lru = 0;
      for (size_t i = 1; i < classes.size(); i++)
        if (classes[i].stamp < classes[lru].stamp) lru = i;
      classes.erase(classes.begin() + lru);
    }
    classes.emplace_back();
    PodClass &c = classes.back();
    c.topo = k;
    c.max_pod = max_pod;
    c.stamp = ++class_clock;
    c.only_pods = true;
    for (int r = 0; r < R; r++)
      if (r == 3 ? max_pod[r] > 1 : max_pod[r] > 0) c.only_pods = false;
    c.cnt.assign(N, 0);
    c.leaf_cnt.assign(topos[k].doms.size(), 0);
    if (!c.only_pods)
      for (int n : topos[k].doms[0].nodes) {
        c.cnt[n] = count_node(max_pod, n);
        for (int d = leaf_of[k][n]; d >= 0; d = topos[k].doms[d].parent) c.leaf_cnt[d] += c.cnt[n];
      }
    return c;
  }
  void subtree_free_live(Topo &tp, int di) {
    Dom &d = tp.doms[di];
    if (d.children.empty()) {
      if (d.level >= 0)
        for (int r = 0; r < R; r++) d.free[r] = d.free_live[r];
      return;
    }
    for (int c : d.children) {
      subtree_free_live(tp, c);
      for (int r = 0; r < R; r++) tp.doms[di].free[r] += tp.doms[c].free[r];
    }
  }
  int subtree_allocatable_live(Topo &tp, int di, const PodClass &c, int n_tasks) {
    Dom &d = tp.doms[di];
    d.alloc_pods = 0;
    if (d.children.empty()) {
      d.alloc_pods = c.only_pods ? n_tasks * (int)d.nodes.size() : c.leaf_cnt[di];
      return d.alloc_pods;
    }
    for (int ch : d.children) {
      int a = subtree_allocatable_live(tp, ch, c, n_tasks);
      tp.doms[di].alloc_pods += a;
    }
    return tp.doms[di].alloc_pods;
  }
  bool any() const {
    for (char c : job_general)
      if (c) return true;
    return false;
  }
  bool constrained(int job) const { return !job_general.empty() && job_general[job]; }
  double avail(int r, int n) const { return mI_(r, n) + mL_(r, n); }

  void build(const kai_snapshot *s) {
    topos.clear();
    live = false;
    classes.clear();
    level_begin.clear();
    node_domain.clear();
    N = s->n_nodes;
    R = s->n_res;
    if (s->n_topologies > 0 && s->topology_level_begin && s->node_domain) {
      level_begin.assign(s->topology_level_begin, s->topology_level_begin + s->n_topologies + 1);
      node_domain.assign(s->node_domain, s->node_domain + (size_t)level_begin.back() * N);
      for (int k = 0; k < s->n_topologies; k++) {
        Topo tp;
        tp.lb = level_begin[k];
        tp.le = level_begin[k + 1];
        tp.doms.emplace_back();
        tp.node_in.assign(N, 0);
        tp.dom_at.assign(tp.le - tp.lb, {});
        for (int l = tp.lb; l < tp.le; l++) {
          int mx = -1;
          for (int n = 0; n < N; n++) mx = std::max(mx, ND(l, n));
          tp.dom_at[l - tp.lb].assign(mx + 1, -1);
        }
        for (int n = 0; n < N; n++) {
          bool in = tp.le > tp.lb;
          for (int l = tp.lb; l < tp.le; l++)
            if (ND(l, n) < 0) in = false;
          if (!in) continue;
          tp.node_in[n] = 1;
          tp.doms[0].nodes.push_back(n);
          int parent = 0;
          for (int l = tp.lb; l < tp.le; l++) {
            int &di = tp.dom_at[l - tp.lb][ND(l, n)];
            if (di < 0) {
              di = (int)tp.doms.size();
              tp.doms.emplace_back();
              tp.doms[di].level = l;
              tp.doms[di].id = ND(l, n);
              tp.doms[di].parent = parent;
              tp.doms[parent].children.push_back(di);
            }
            tp.doms[di].nodes.push_back(n);
            parent = di;
          }
        }
        for (auto &d : tp.doms)
          std::sort(d.children.begin(), d.children.end(), [&](int a, int b) { return tp.doms[a].id < tp.doms[b].id; });
        topos.push_back(tp);
      }
    }
    {
      const int NJ = s->n_jobs, NS = s->n_podsets;
      set_parent.clear();
      set_rank.clear();
      set_con.clear();
      job_root_set.assign(NJ, -1);
      ps_set.assign(NS, -1);
      ps_con.assign(NS, std::array<int, 3>{-1, -1, -1});
      std::vector<int> ps_job(NS, -1);
      for (int j = 0; j < NJ; j++)
        for (int ps = s->job_podset_begin[j]; ps < s->job_podset_begin[j + 1]; ps++) ps_job[ps] = j;
      if (s->job_sgs_begin && s->sgs_parent && s->podset_sgs) {
        for (int g = 0; g < s->n_subgroup_sets; g++) {
          set_parent.push_back(s->sgs_parent[g]);
          set_rank.push_back(s->sgs_name_rank ? s->sgs_name_rank[g] : g);
          set_con.push_back({s->sgs_topology ? s->sgs_topology[g] : -1, s->sgs_required_level ? s->sgs_required_level[g] : -1,
                             s->sgs_preferred_level ? s->sgs_preferred_level[g] : -1});
        }
        for (int j = 0; j < NJ; j++) job_root_set[j] = s->job_sgs_begin[j];
        for (int ps = 0; ps < NS; ps++) {
          ps_set[ps] = s->podset_sgs[ps];
          if (s->podset_topology)
            ps_con[ps] = {s->podset_topology[ps], s->podset_required_level ? s->podset_required_level[ps] : -1,
                          s->podset_preferred_level ? s->podset_preferred_level[ps] : -1};
        }
      } else {
        for (int j = 0; j < NJ; j++) {
          job_root_set[j] = (int)set_parent.size();
          set_parent.push_back(-1);
          set_rank.push_back(0);
          set_con.push_back({s->job_topology ? s->job_topology[j] : -1, s->job_required_level ? s->job_required_level[j] : -1,
                             s->job_preferred_level ? s->job_preferred_level[j] : -1});
          for (int ps = s->job_podset_begin[j]; ps < s->job_podset_begin[j + 1]; ps++) ps_set[ps] = job_root_set[j];
        }
      }
      const int G = (int)set_parent.size();
      set_children.assign(G, {});
      set_podsets.assign(G, {});
      for (int g = 0; g < G; g++)
        if (set_parent[g] >= 0) set_children[set_parent[g]].push_back(g);
      for (auto &ch : set_children) std::sort(ch.begin(), ch.end(), [&](int a, int b) { return set_rank[a] < set_rank[b]; });
      for (int ps = 0; ps < NS; ps++)
        if (ps_set[ps] >= 0) set_podsets[ps_set[ps]].push_back(ps);
      job_general.assign(NJ, 0);
      std::vector<int> job_of_root(G, -1);
      for (int j = 0; j < NJ; j++)
        if (job_root_set[j] >= 0) job_of_root[job_root_set[j]] = j;
      for (int g = 0; g < G; g++) {
        if (set_con[g][0] == -1 && set_parent[g] < 0) continue;
        int root = g;
        while (set_parent[root] >= 0) root = set_parent[root];
        if (job_of_root[root] >= 0) job_general[job_of_root[root]] = 1;
      }
      for (int ps = 0; ps < NS; ps++)
        if (ps_con[ps][0] != -1 && ps_job[ps] >= 0) job_general[ps_job[ps]] = 1;
    }
  }

  // job_filtering.go:445-486 getJobRatioToFreeResources (Quantity.Value() of a milli quantity rounds up)
  double job_ratio_to_free(const double *tasks_res, const Dom &d) const {
    double ratio = 0.0;
    bool empty = true;
    for (int r = 0; r < R; r++)
      if (tasks_res[r] > 0) empty = false;
    if (empty) return 0.0;
    if (tasks_res[KAI_RES_GPU] > 0) ratio = std::max(ratio, tasks_res[KAI_RES_GPU] / d.free[KAI_RES_GPU]);
    for (int r = 0; r < R; r++) {
      if (r == KAI_RES_GPU || r == 3) continue;
      int64_t tq = r == KAI_RES_MEM ? (int64_t)tasks_res[r] : (int64_t)std::ceil((double)(int64_t)tasks_res[r] / 1000.0);
      if (tq == 0) continue;
      int64_t fq = r == KAI_RES_MEM ? (int64_t)d.free[r] : (int64_t)std::ceil((double)(int64_t)d.free[r] / 1000.0);
      double rr = fq == 0 ? 1000.0 : (double)tq / (double)fq;
      ratio = std::max(ratio, rr);
    }
    return ratio;
  }
  bool domain_fit(const double *tasks_res, int tasks_count, const Dom &d) const {  // :302-320 checkJobDomainFit
    if (d.alloc_pods != -1) return d.alloc_pods >= tasks_count;
    return !(job_ratio_to_free(tasks_res, d) > 1.0);
  }
  // getJobRatioToFreeResources memo: the ratio of a (job resource sum, domain) pair changes only when the domain's
  // free resources do; `ver` counts those changes (node_changed walks the ancestors)
  struct RatioClass {
    std::vector<double> tasks_res;
    int topo = -1;
    std::vector<double> ratio;
    std::vector<unsigned int> ver;
  };
  std::vector<RatioClass> ratio_classes;
  std::vector<std::vector<unsigned int>> dom_ver;  // [topology][dom], starts at 1
  RatioClass *cur_ratio = nullptr;
  void select_ratio_class(int k, const double *tasks_res) {
    for (RatioClass &c : ratio_classes)
      if (c.topo == k && std::equal(c.tasks_res.begin(), c.tasks_res.end(), tasks_res)) {
        cur_ratio = &c;
        return;
      }
    if (ratio_classes.size() >= 64) ratio_classes.erase(ratio_classes.begin());
    ratio_classes.emplace_back();
    RatioClass &c = ratio_classes.back();
    c.topo = k;
    c.tasks_res.assign(tasks_res, tasks_res + R);
    c.ratio.assign(topos[k].doms.size(), 0.0);
    c.ver.assign(topos[k].doms.size(), 0u);
    cur_ratio = &c;
  }
  double cached_ratio(int k, const double *tasks_res, int di) {
    RatioClass &c = *cur_ratio;
    const unsigned int v = dom_ver[k][di];
    if (c.ver[di] != v) {
      c.ratio[di] = job_ratio_to_free(tasks_res, topos[k].doms[di]);
      c.ver[di] = v;
    }
    return c.ratio[di];
  }
  void sort_tree(Topo &tp, int di, const double *tasks_res, int max_depth_level) {  // :396-420
    std::vector<std::pair<double, int>> keyed;
    const int kk = (int)(&tp - &topos[0]);
    for (int c : tp.doms[di].children) keyed.push_back({cached_ratio(kk, tasks_res, c), c});
    std::stable_sort(keyed.begin(), keyed.end(), [&](const std::pair<double, int> &a, const std::pair<double, int> &b) {
      if (a.first != b.first) return a.first > b.first;
      return tp.doms[a.second].id < tp.doms[b.second].id;
    });
    for (size_t i = 0; i < keyed.size(); i++) tp.doms[di].children[i] = keyed[i].second;
    if (tp.doms[di].level == max_depth_level) return;
    std::vector<int> ch = tp.doms[di].children;
    for (int c : ch) sort_tree(tp, c, tasks_res, max_depth_level);
  }
  void level_domains(const Topo &tp, int di, int level, std::vector<int> &out) const {
    if (tp.doms[di].level == level) {
      out.push_back(di);
      return;
    }
    for (int c : tp.doms[di].children) level_domains(tp, c, level, out);
  }

  struct Result {
    bool ok = true;            // false: configuration error (the job fails)
    bool passthrough = false;  // no constraint (or no tasks): the node set is handed on unchanged
    int topo = -1;
    std::vector<int> domains;  // candidate domains (indices into topos[topo].doms), in the order to try
    int pref_level = -1;       // global level index when node scores apply
    std::vector<std::pair<int, int>> scores;  // (domain id at the preferred level, bucket 0..10)
  };
  // subSetNodesFn for the job's root SubGroupSet.  `in_set(n)`: the node set handed to allocate (all nodes, or the
  // solver's feasible set).  `active_nodes`: nodes of the job's active-allocated pods; has_active: any podset of the
  // (view of the) job counts active-allocated pods.
  // `base_nodes`: the nodes of the innermost domain already selected further up the SubGroupSet tree (or null = all).
  Result subset(const std::array<int, 3> &con, const std::vector<int> &tasks, const std::vector<int> *base_nodes,
                const std::function<bool(int)> &in_set, bool has_active, const std::vector<int> &active_nodes,
                bool all_nodes = false) {
    Result res;
    const int k = con[0];
    if (k == -2) return res;  // requested topology does not exist: no node set
    if (k < 0 || tasks.empty()) {
      res.passthrough = true;
      return res;
    }
    Topo &tp = topos[k];
    res.topo = k;
    const int req = con[1], pref = con[2];
    // common.go:17-61 lowestCommonDomainID over nodeSet ∩ topology nodes
    int dom = 0;
    {
      int first = -1;
      std::vector<char> all(tp.le - tp.lb, 1);
      std::vector<int> value(tp.le - tp.lb, -1);
      for (int n : (base_nodes ? *base_nodes : tp.doms[0].nodes)) {
        if (base_nodes && !tp.node_in[n]) continue;
        if (all_nodes && first >= 0) {  // every topology node is in the set: only "all equal?" per level matters
          if ((int)tp.lcd_all.size() == tp.le - tp.lb) {
            all = tp.lcd_all;
            break;
          }
        }
        if (!all_nodes && !in_set(n)) continue;
        if (first < 0) {
          first = n;
          for (int l = tp.lb; l < tp.le; l++) value[l - tp.lb] = ND(l, n);
        } else {
          for (int l = tp.lb; l < tp.le; l++)
            if (ND(l, n) != value[l - tp.lb]) all[l - tp.lb] = 0;
        }
      }
      if (all_nodes && first >= 0 && (int)tp.lcd_all.size() != tp.le - tp.lb) tp.lcd_all = all;  // computed once per load
      for (int l = tp.lb; l < tp.le && first >= 0; l++) {
        if (!all[l - tp.lb]) break;
        dom = tp.dom_at[l - tp.lb][value[l - tp.lb]];
        if (pref >= 0 && l - tp.lb == pref) break;
      }
    }
    // gather what checkJobDomainFit(domain) needs first: when the lowest common domain cannot take the job (a full
    // cluster's tail of pending gangs) nothing below has to be evaluated
    ensure_live();
    double tasks_res0[KAI_MAX_RES] = {0};
    std::vector<double> max_pod0(R, 0.0);
    int gpu_pods0 = 0;
    for (int t : tasks) {
      if (t_req[(size_t)t * R + KAI_RES_GPU] > 0) gpu_pods0++;
      for (int r = 0; r < R; r++) {
        tasks_res0[r] += t_req[(size_t)t * R + r];
        max_pod0[r] = std::max(max_pod0[r], t_req[(size_t)t * R + r]);
      }
    }
    {
      bool uniform = true;
      for (int r = 3; r < R; r++) {
        int c = 0;
        for (int t : tasks)
          if (t_req[(size_t)t * R + r] != 0) c++;
        if (c != 0 && c != (int)tasks.size()) uniform = false;
      }
      Dom probe = Dom();
      for (int r = 0; r < R; r++) probe.free[r] = tp.doms[dom].free_live[r];
      if ((gpu_pods0 == (int)tasks.size() || gpu_pods0 == 0) && uniform) {
        PodClass &pc = pod_class(k, max_pod0);
        probe.alloc_pods = pc.only_pods ? (int)tasks.size() * (int)tp.doms[dom].nodes.size() : pc.leaf_cnt[dom];
      }
      if (!domain_fit(tasks_res0, (int)tasks.size(), probe)) return res;
    }
    for (auto &d : tp.doms) {  // treeAllocatableCleanup
      d.alloc_pods = -1;
      for (int r = 0; r < KAI_MAX_RES; r++) d.free[r] = 0;
    }
    ensure_live();
    subtree_free_live(tp, dom);
    int gpu_pods = 0;
    for (int t : tasks)
      if (t_req[(size_t)t * R + KAI_RES_GPU] > 0) gpu_pods++;
    bool scalars_uniform = true;
    for (int r = 3; r < R; r++) {
      int c = 0;
      for (int t : tasks)
        if (t_req[(size_t)t * R + r] != 0) c++;
      if (c != 0 && c != (int)tasks.size()) scalars_uniform = false;
    }
    if ((gpu_pods == (int)tasks.size() || gpu_pods == 0) && scalars_uniform) {  // useRepresentorPodsAccounting
      std::vector<double> max_pod(R, 0.0);
      for (int t : tasks)
        for (int r = 0; r < R; r++) max_pod[r] = std::max(max_pod[r], t_req[(size_t)t * R + r]);
      subtree_allocatable_live(tp, dom, pod_class(k, max_pod), (int)tasks.size());
    }
    double tasks_res[KAI_MAX_RES] = {0};
    for (int t : tasks)
      for (int r = 0; r < R; r++) tasks_res[r] += t_req[(size_t)t * R + r];
    const int tasks_count = (int)tasks.size();
    if (!domain_fit(tasks_res, tasks_count, tp.doms[dom])) return res;
    if (req == -2 || pref == -2 || (req < 0 && pref < 0)) {
      res.ok = false;
      return res;
    }
    select_ratio_class(k, tasks_res);
    sort_tree(tp, dom, tasks_res, pref >= 0 ? tp.lb + pref : tp.lb + req);
    if (pref >= 0) {  // node_scoring.go:36-53
      res.pref_level = tp.lb + pref;
      std::vector<int> lvl;
      level_domains(tp, dom, tp.lb + pref, lvl);
      for (size_t i = 0; i < lvl.size(); i++) {
        double score = ((double)(i + 1) / (double)lvl.size()) * 10;
        res.scores.push_back({tp.doms[lvl[i]].id, (int)std::floor(score)});
      }
    }
    std::vector<int> relevant;
    {
      bool found_pref = false, found_req = false;
      for (int l = tp.le - 1; l >= tp.lb - 1; l--) {
        int li = l >= tp.lb ? l - tp.lb : -1;
        if (l >= tp.lb && pref >= 0 && li == pref) found_pref = true;
        if (l >= tp.lb && req >= 0 && li == req) found_req = true;
        if (found_pref || found_req) relevant.push_back(l >= tp.lb ? l : -1);
        if (found_req) break;
      }
    }
    std::vector<char> allowed(tp.doms.size(), 1);
    if (has_active && req >= 0) {  // :269-300 getRelevantDomainsWithAllocatedPods
      std::fill(allowed.begin(), allowed.end(), 0);
      std::function<void(int)> mark = [&](int di) {
        allowed[di] = 1;
        for (int c : tp.doms[di].children) mark(c);
      };
      for (int n : active_nodes)
        if (n >= 0 && tp.node_in[n]) mark(tp.dom_at[req][ND(tp.lb + req, n)]);
    }
    std::vector<char> chosen(tp.doms.size(), 0);
    bool any_dom = false;
    for (int l : relevant)
      for (size_t di = 0; di < tp.doms.size(); di++) {
        if (tp.doms[di].level != l || !allowed[di]) continue;
        if (!domain_fit(tasks_res, tasks_count, tp.doms[di])) continue;
        chosen[di] = 1;
        any_dom = true;
      }
    if (!any_dom) return res;
    std::vector<std::vector<int>> levels;  // sortDomainInfos: reverse level order of the sorted tree
    std::vector<int> cur{0};
    while (!cur.empty()) {
      levels.push_back(cur);
      std::vector<int> next;
      for (int di : cur)
        for (int c : tp.doms[di].children) next.push_back(c);
      cur = next;
    }
    for (int li = (int)levels.size() - 1; li >= 0; li--)
      for (int di : levels[li])
        if (chosen[di]) res.domains.push_back(di);
    return res;
  }

  // ---- GPU side: select a domain as the row set of the following sweeps; publish / clear the score table ----
  void select_domain(Seq &seq, int topo, int di, int slot) const {
    const Topo &tp = topos[topo];
    const Dom &d = tp.doms[di];
    if (d.level < 0)
      emit_ext(seq, EXT_SELECT_ROOT, (unsigned int)(tp.lb | (tp.le << 8) | (slot << 16)), 0);
    else
      emit_ext(seq, EXT_SELECT, (unsigned int)((d.level + 1) | (slot << 8)), (unsigned int)d.id);
  }
  bool node_in_domain(int topo, int di, int n) const {
    const Topo &tp = topos[topo];
    const Dom &d = tp.doms[di];
    if (!tp.node_in[n]) return false;
    return d.level < 0 || ND(d.level, n) == d.id;
  }
  // The scanners keep the per-domain bucket table between jobs; the host remembers what they hold and sends only the
  // entries that differ (consecutive gangs sort the racks almost identically).  scores_off() before any sweep of a job
  // without node scores.
  int gpu_pref_level = -1;
  std::vector<unsigned char> gpu_bucket;   // what the scanners hold (255 = no entry)
  std::vector<int> gpu_set;                // domain ids with an entry
  bool push_scores(Seq &seq, const Result &r) {  // false: more preferred-level domains than the table holds
    if (r.pref_level < 0) {
      scores_off(seq);
      return true;
    }
    if (gpu_bucket.empty()) gpu_bucket.assign(kDomBuckets, 255);
    if (gpu_pref_level != r.pref_level) {
      emit_ext(seq, EXT_SCORE_BEGIN, (unsigned int)r.pref_level, 0);
      for (int d : gpu_set) gpu_bucket[d] = 255;
      gpu_set.clear();
      gpu_pref_level = r.pref_level;
    }
    std::vector<unsigned char> want_mark;
    for (auto &kv : r.scores)
      if (kv.first >= kDomBuckets) return false;
    // entries to drop: held by the scanners, absent from the new table
    std::vector<int> keep;
    {
      std::vector<char> in_new(kDomBuckets, 0);
      for (auto &kv : r.scores) in_new[kv.first] = 1;
      for (int d : gpu_set) {
        if (in_new[d]) {
          keep.push_back(d);
        } else {
          emit_ext(seq, EXT_SCORE, (unsigned int)d, 255u);
          gpu_bucket[d] = 255;
        }
      }
    }
    gpu_set = keep;
    for (auto &kv : r.scores) {
      if (gpu_bucket[kv.first] == (unsigned char)kv.second) continue;
      if (gpu_bucket[kv.first] == 255) gpu_set.push_back(kv.first);
      emit_ext(seq, EXT_SCORE, (unsigned int)kv.first, (unsigned int)kv.second);
      gpu_bucket[kv.first] = (unsigned char)kv.second;
    }
    return true;
  }
  void scores_off(Seq &seq) {
    if (gpu_pref_level < 0) return;
    emit_ext(seq, EXT_SCORE_END, 0, 0);
    for (int d : gpu_set) gpu_bucket[d] = 255;
    gpu_set.clear();
    gpu_pref_level = -1;
  }
  void reset_gpu_state() {  // a new action starts with scoring off and an undefined table
    gpu_pref_level = -1;
    gpu_set.clear();
    if (!gpu_bucket.empty()) std::fill(gpu_bucket.begin(), gpu_bucket.end(), 255);
  }
};

// allocate.go:36-83 allocateSubGroupSet / allocateSubGroupSetOnNodes / allocatePodSet over the SubGroupSet tree of a
// job, shared by the allocate action (live job) and the solver's simulations (views).  Ops supplies the session side:
//   int  active_alloc(int ps);  void active_nodes(int ps, std::vector<int>&);  bool podset_less(int a, int b);
//   int  checkpoint();  void rollback(int cp);  bool place(const std::vector<int> &tasks, unsigned int xbits);
//   bool extra_in_set(int n);  bool all_nodes();
template <class Ops>
struct TopoAllocator {
  TopologyHost &th;
  Seq &seq;
  Ops &ops;
  int job;
  std::map<int, TopologyHost::Result> tables;  // subGroupNodeScores of this AllocateJob: key = set id or G + podset id
  std::vector<std::pair<int, int>> stack;      // (topology, domain) selected on the way down; slot = position
  bool unsupported = false;

  TopoAllocator(TopologyHost &t, Seq &s, Ops &o, int j) : th(t), seq(s), ops(o), job(j) {}
  void podsets_under(int g, std::vector<int> &out) const {
    for (int ps : th.set_podsets[g]) out.push_back(ps);
    for (int c : th.set_children[g]) podsets_under(c, out);
  }
  bool in_set(int n) const {
    for (auto &e : stack)
      if (!th.node_in_domain(e.first, e.second, n)) return false;
    return ops.extra_in_set(n);
  }
  TopologyHost::Result subset(const std::array<int, 3> &con, const std::vector<int> &under, const std::vector<int> &tasks) {
    bool has_active = false;
    std::vector<int> act;
    for (int ps : under) {
      if (ops.active_alloc(ps) > 0) has_active = true;
      ops.active_nodes(ps, act);
    }
    const std::vector<int> *base = stack.empty() ? nullptr : &th.topos[stack.back().first].doms[stack.back().second].nodes;
    return th.subset(con, tasks, base, [&](int n) { return in_set(n); }, has_active, act, stack.empty() && ops.all_nodes());
  }
  // runs `body` once per candidate domain until it succeeds
  template <class Body>
  bool over_domains(const TopologyHost::Result &r, Body body) {
    if (!r.ok) return false;
    if (r.passthrough) return body();
    if (r.domains.empty()) return false;
    if ((int)stack.size() >= kDomSlots) {
      unsupported = true;
      return false;
    }
    for (int di : r.domains) {
      const int cp = ops.checkpoint();
      stack.push_back({r.topo, di});
      th.select_domain(seq, r.topo, di, (int)stack.size() - 1);
      const bool ok = body();
      stack.pop_back();
      if (ok) return true;
      if (unsupported) return false;
      ops.rollback(cp);
    }
    return false;
  }
  bool alloc_set(int g, const std::vector<int> &tasks) {
    std::vector<int> under;
    podsets_under(g, under);
    TopologyHost::Result r = subset(th.set_con[g], under, tasks);
    if (r.ok && !r.passthrough && r.pref_level >= 0) tables[g] = r;
    return over_domains(r, [&]() { return set_on_nodes(g, tasks); });
  }
  bool set_on_nodes(int g, const std::vector<int> &tasks) {
    for (int c : th.set_children[g]) {  // orderedSubGroupSets: by name
      std::vector<int> under, sub;
      podsets_under(c, under);
      for (int t : tasks)
        for (int ps : under)
          if (th.t_podset[t] == ps) sub.push_back(t);
      if (!alloc_set(c, sub)) return false;
    }
    std::vector<int> own = th.set_podsets[g];  // orderedPodSets
    std::sort(own.begin(), own.end(), [&](int a, int b) { return ops.podset_less(a, b); });
    for (int ps : own) {
      std::vector<int> pt;
      for (int t : tasks)
        if (th.t_podset[t] == ps) pt.push_back(t);
      TopologyHost::Result r = subset(th.ps_con[ps], {ps}, pt);
      const int key = (int)th.set_parent.size() + ps;
      if (r.ok && !r.passthrough && r.pref_level >= 0) tables[key] = r;
      if (!over_domains(r, [&]() { return place_podset(ps, pt); })) return false;
    }
    return true;
  }
  bool place_podset(int ps, const std::vector<int> &pt) {
    if (pt.empty()) return true;
    // getRelevantNodeScores: the PodSet's own table, else the nearest ancestor set's
    const TopologyHost::Result *tab = nullptr;
    auto it = tables.find((int)th.set_parent.size() + ps);
    if (it != tables.end()) tab = &it->second;
    for (int g = th.ps_set[ps]; !tab && g >= 0; g = th.set_parent[g]) {
      it = tables.find(g);
      if (it != tables.end()) tab = &it->second;
    }
    if (tab) {
      if (!th.push_scores(seq, *tab)) {
        unsupported = true;
        return false;
      }
    } else {
      th.scores_off(seq);
    }
    const unsigned int xbits = stack.empty() ? 0u : (XB_RESTRICT_DOM | ((unsigned int)stack.size() << 8));
    return ops.place(pt, xbits);
  }
};

}  // namespace kai
