"""Parity of the CUDA engine with the CPU oracle through the C ABI (GPU box only).

Bit-exact: bindings (task -> node), task statuses, job visiting order and outcomes, node Idle/Releasing
tables, queue Allocated / Request / totals.  Fair shares are compared within 1e-6 here; the inputs of this module are
integer valued, so every sum is exact in any order and these tests cannot tell a summation order from another.
test_value_regime_gpu.py runs non-round values (inexact totals and queue sums, score near-ties, fractional fair shares)
with every table, the fair shares included, compared bit for bit.
"""
import os

import numpy as np
import pytest

import dsl
from fixtures import action_cases, case_config
from kai_scheduler_b200 import abi, synthetic
from kai_scheduler_b200.engine import Engine
from oracle_lib import Oracle

pytestmark = pytest.mark.gpu

ALLOCATE = action_cases(["allocate__"], single_action="allocate")


def assert_same(res_e: abi.Result, res_o: abi.Result):
    np.testing.assert_array_equal(res_e.task_node, res_o.task_node)
    np.testing.assert_array_equal(res_e.task_status, res_o.task_status)
    np.testing.assert_array_equal(res_e.visits, res_o.visits)
    np.testing.assert_array_equal(res_e.node_idle, res_o.node_idle)
    np.testing.assert_array_equal(res_e.node_releasing, res_o.node_releasing)
    np.testing.assert_array_equal(res_e.queue_allocated, res_o.queue_allocated)
    np.testing.assert_array_equal(res_e.queue_allocated_non_preemptible, res_o.queue_allocated_non_preemptible)
    np.testing.assert_array_equal(res_e.queue_request, res_o.queue_request)
    np.testing.assert_array_equal(res_e.total_resource, res_o.total_resource)
    # DRF / fair shares: BASELINE.json tolerance 1e-6; integer-valued inputs give exact equality
    np.testing.assert_allclose(res_e.queue_fair_share, res_o.queue_fair_share, rtol=0, atol=1e-6)
    assert res_e.pods_placed == res_o.pods_placed


def run_both(snap, action="allocate", cfg=None):
    e = Engine(cfg)
    e.load(snap)
    re_ = e.run(action)
    e.close()
    o = Oracle(cfg)
    o.load(snap)
    ro = o.run(action)
    return re_, ro


@pytest.mark.parametrize("cid,case", ALLOCATE, ids=[c[0] for c in ALLOCATE])
def test_allocate_tables_gpu(cid, case):
    snap, meta = dsl.build_snapshot(case["topology"])
    re_, ro = run_both(snap, cfg=case_config(case))
    assert_same(re_, ro)
    errs = dsl.check_expectations(case["topology"], meta, re_, snap)
    assert not errs, f"{case['source']} #{case['index']}: {errs}"


SOLVER = (action_cases(["reclaim__"], single_action="reclaim") + action_cases(["consolidation__"], single_action="consolidation")
          + action_cases(["preempt__"], single_action="preempt"))


@pytest.mark.parametrize("cid,case", SOLVER, ids=[c[0] for c in SOLVER])
def test_solver_tables_gpu(cid, case):
    """reclaim / consolidation: victim sets, moved victims and preemptor bindings against the oracle AND the
    reference's expectations (65 + 24 tables)."""
    snap, meta = dsl.build_snapshot(case["topology"])
    re_, ro = run_both(snap, action=case["actions"][0])
    assert_same(re_, ro)
    assert re_.pods_evicted == ro.pods_evicted
    errs = dsl.check_expectations(case["topology"], meta, re_, snap)
    assert not errs, f"{case['source']} #{case['index']}: {errs}"


INTEGRATION = action_cases(["integration_tests__"])


@pytest.mark.parametrize("cid,case", INTEGRATION, ids=[c[0] for c in INTEGRATION])
def test_integration_tables_gpu(cid, case):
    """The reference's multi-action, multi-round integration tables through the engine: allocate, consolidation,
    reclaim, preempt, stalegangeviction on one session per round; expectations of the reference + every round's
    final state equal to the oracle's."""
    import copy
    e_case, o_case = copy.deepcopy(case), copy.deepcopy(case)
    seen = {"e": [], "o": []}

    class Tap:
        def __init__(self, inner, key):
            self.inner, self.key = inner, key

        def load(self, snap):
            self.inner.load(snap)

        def run(self, action):
            r = self.inner.run(action)
            seen[self.key].append((r.task_status.copy(), r.task_node.copy(), r.node_idle.copy(), r.queue_allocated.copy()))
            return r

        def close(self):
            if hasattr(self.inner, "close"):
                self.inner.close()

    errs = dsl.run_integration_case(e_case, lambda: Tap(Engine(), "e"))
    assert not errs, f"{case['source']} #{case['index']}: {errs[:3]}"
    dsl.run_integration_case(o_case, lambda: Tap(Oracle(), "o"))
    assert len(seen["e"]) == len(seen["o"])
    for a, b in zip(seen["e"], seen["o"]):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("kw", [
    dict(n_nodes=10), dict(n_nodes=50), dict(n_nodes=100),          # BenchmarkReclaimLargeJobs_{10,50,100}Node
    dict(n_nodes=40, victim_queues=3, reclaimer_jobs=6, reclaimer_tasks=2, reclaimer_gpus=4.0),  # config-5 shape
    dict(n_nodes=64, running_per_node=6, victim_queues=2, reclaimer_jobs=20, reclaimer_tasks=1, reclaimer_gpus=2.0),
])
@pytest.mark.parametrize("action", ["reclaim", "consolidation"])
def test_solver_synthetic(kw, action):
    snap = synthetic.reclaim_snapshot(**kw)
    re_, ro = run_both(snap, action=action)
    assert_same(re_, ro)
    assert re_.pods_evicted == ro.pods_evicted


@pytest.mark.parametrize("kw", [
    dict(n_nodes=512, n_gangs=60, nodes_per_rack=8, racks_per_leaf=4, leaves_per_spine=4, running_fraction=0.3),
    dict(n_nodes=300, n_gangs=50, nodes_per_rack=5, racks_per_leaf=3, leaves_per_spine=2, running_fraction=0.5, max_pods=6),
    dict(n_nodes=4096, n_gangs=600),  # config4-small: 16 nodes / rack, 16 racks / leaf
])
def test_topology_synthetic(kw):
    """BASELINE config 4 shape: 3-tier topology, node-exclusive gangs, required leaf|rack + preferred rack."""
    snap = synthetic.topology_snapshot(**kw)
    re_, ro = run_both(snap)
    assert_same(re_, ro)
    assert re_.pods_placed > 0


def test_topology_cycle_with_solver():
    """topology-constrained pending gangs through consolidation / reclaim simulations as well"""
    snap = synthetic.topology_snapshot(n_nodes=96, n_gangs=20, nodes_per_rack=4, racks_per_leaf=3, leaves_per_spine=2,
                                       running_fraction=0.6, max_pods=4)
    e = Engine()
    e.load(snap)
    o = Oracle()
    o.load(snap)
    for action in ("allocate", "consolidation", "reclaim", "preempt"):
        re_, ro = e.run(action), o.run(action)
        assert_same(re_, ro)
    e.close()


@pytest.mark.parametrize("action", ["reclaim", "consolidation"])
def test_solver_scheduling_signatures(action):
    """UseSchedulingSignatures = true (production default): jobs not easier than a failed representative are skipped."""
    snap = synthetic.reclaim_snapshot(n_nodes=24, running_per_node=8, victim_queues=2, reclaimer_jobs=30,
                                      reclaimer_tasks=2, reclaimer_gpus=5.0)
    snap.job_signature = np.where(snap.job_queue == 2, 7, -1).astype(np.int32)
    cfg = abi.make_config(use_scheduling_signatures=True)
    re_, ro = run_both(snap, action=action, cfg=cfg)
    assert_same(re_, ro)
    re2, _ = run_both(snap, action=action)
    assert len(re_.visits) <= len(re2.visits)


def test_full_cycle_allocate_consolidation_reclaim():
    """One scheduling cycle: the three actions in the default order on ONE session (state carries over)."""
    snap = synthetic.reclaim_snapshot(n_nodes=48, running_per_node=7, victim_queues=2, reclaimer_jobs=12,
                                      reclaimer_tasks=2, reclaimer_gpus=3.0)
    e = Engine()
    e.load(snap)
    o = Oracle()
    o.load(snap)
    for action in ("allocate", "consolidation", "reclaim", "preempt"):
        re_, ro = e.run(action), o.run(action)
        assert_same(re_, ro)
        assert re_.pods_evicted == ro.pods_evicted
    e.close()


@pytest.mark.parametrize("grid,env", [("2", None), ("5", "KAI_NO_TOPM"), ("148", None), ("148", "KAI_NO_BATCHING")])
def test_solver_tables_forced_grid(grid, env, monkeypatch):
    monkeypatch.setenv("KAI_GRID_EXACT", grid)
    if env:
        monkeypatch.setenv(env, "1")
    for cid, case in SOLVER:
        snap, meta = dsl.build_snapshot(case["topology"])
        re_, ro = run_both(snap, action=case["actions"][0])
        assert_same(re_, ro)


@pytest.mark.parametrize("grid", ["2", "3", "148"])
def test_allocate_tables_forced_grid(grid, monkeypatch):
    """Same tables with forced CTA counts (including scanners that own no node)."""
    monkeypatch.setenv("KAI_GRID_EXACT", grid)
    for cid, case in ALLOCATE:
        snap, meta = dsl.build_snapshot(case["topology"])
        re_, ro = run_both(snap, cfg=case_config(case))
        assert_same(re_, ro)


@pytest.mark.parametrize("kw", [
    dict(n_nodes=100, n_jobs=500, tasks_per_job=1, n_queues=10),            # BASELINE config 1
    dict(n_nodes=64, n_jobs=700, tasks_per_job=1, n_queues=4),              # over-subscribed: failures + leftovers
    dict(n_nodes=300, n_jobs=400, tasks_per_job=4, n_queues=12),            # gangs, many queues
    dict(n_nodes=257, n_jobs=600, tasks_per_job=3, n_queues=7, mixed=True),  # request mix, ragged sizes
    dict(n_nodes=1000, n_jobs=3000, tasks_per_job=2, n_queues=40, mixed=True),
])
def test_synthetic_parity(kw):
    snap = synthetic.benchmark_snapshot(**kw)
    re_, ro = run_both(snap)
    assert_same(re_, ro)


@pytest.mark.parametrize("env", [("KAI_NO_BATCHING", "1"), ("KAI_NO_TOPM", "1")])
def test_synthetic_parity_fallback_paths(env, monkeypatch):
    """Same answers with batching off, and with single-candidate answers (no top-M lists)."""
    monkeypatch.setenv(env[0], env[1])
    for kw in (dict(n_nodes=300, n_jobs=400, tasks_per_job=4, n_queues=12),
               dict(n_nodes=257, n_jobs=600, tasks_per_job=3, n_queues=7, mixed=True)):
        snap = synthetic.benchmark_snapshot(**kw)
        re_, ro = run_both(snap)
        assert_same(re_, ro)


def test_batching_reduces_sweeps():
    snap = synthetic.benchmark_snapshot(n_nodes=200, n_jobs=1000, tasks_per_job=1, n_queues=4)
    e = Engine()
    e.load(snap)
    res = e.run("allocate")
    st = e.stats()
    e.close()
    assert res.pods_placed == 1000
    assert st.decisions < 400  # 8 identical 1-GPU pods per node fill: about one sweep per node


def test_spread_strategy():
    snap = synthetic.benchmark_snapshot(n_nodes=50, n_jobs=200, tasks_per_job=2, n_queues=4, mixed=True)
    cfg = abi.make_config(gpu_placement=abi.PLACEMENT_SPREAD, cpu_placement=abi.PLACEMENT_SPREAD)
    re_, ro = run_both(snap, cfg=cfg)
    assert_same(re_, ro)


def test_cpu_only_pods_and_cpu_nodes():
    snap = synthetic.benchmark_snapshot(n_nodes=40, n_jobs=300, tasks_per_job=1, n_queues=4)
    # half of the nodes lose their GPUs, a third of the jobs become CPU-only
    snap.node_allocatable[2, ::2] = 0
    snap.node_idle[2, ::2] = 0
    snap.task_req[::3, 2] = 0
    snap.task_req[::3, 0] = 3000
    re_, ro = run_both(snap)
    assert_same(re_, ro)


def test_predicate_mask_and_nominated_node():
    snap = synthetic.benchmark_snapshot(n_nodes=96, n_jobs=200, tasks_per_job=1, n_queues=4)
    rng = np.random.default_rng(7)
    words = (96 + 31) // 32
    mask = rng.integers(0, 2**32, size=(3, words), dtype=np.uint64).astype(np.uint32)
    snap.pred_mask = mask
    snap.task_pred_class = rng.integers(-1, 3, size=snap.n_tasks).astype(np.int32)
    snap.task_nominated = np.where(rng.random(snap.n_tasks) < 0.2, rng.integers(0, 96, size=snap.n_tasks), -1).astype(np.int32)
    re_, ro = run_both(snap)
    assert_same(re_, ro)


def test_empty_and_degenerate_snapshots():
    # no jobs at all
    snap = synthetic.benchmark_snapshot(n_nodes=5, n_jobs=0, tasks_per_job=1, n_queues=4)
    re_, ro = run_both(snap)
    assert_same(re_, ro)
    # a single node, more demand than supply
    snap = synthetic.benchmark_snapshot(n_nodes=1, n_jobs=20, tasks_per_job=1, n_queues=4)
    re_, ro = run_both(snap)
    assert_same(re_, ro)
    assert re_.pods_placed == 8


def test_config2_full_size_properties():
    """BASELINE config 2 at full size: size-independent properties (the oracle needs ~5 s here, so also compare)."""
    snap = synthetic.config_snapshot("config2")
    e = Engine()
    e.load(snap)
    res = e.run("allocate")
    st = e.stats()
    e.close()
    assert res.pods_placed == 40_000
    assert (res.task_node >= 0).all() and (res.task_status == abi.POD_BINDING).all()
    used = np.bincount(res.task_node, minlength=snap.n_nodes)
    assert used.max() <= 8 and (res.node_idle[2] == 8 - used).all()
    # binpack: exactly 5000 nodes completely full, and they are the 5000 lexicographically smallest names
    full = np.nonzero(used == 8)[0]
    assert len(full) == 5000 and set(snap.node_name_rank[full]) == set(range(5000))
    assert 0 < st.decisions <= 40_000  # sweeps; same-node batching places the rest without a sweep
    o = Oracle(threads=min(16, os.cpu_count() or 1))
    o.load(snap)
    ro = o.run("allocate")
    assert_same(res, ro)


def test_fractional_gpu_requests_are_refused_gpu():
    from kai_scheduler_b200.engine import EngineError
    snap = synthetic.benchmark_snapshot(4, 3, n_queues=1)
    snap.task_req = snap.task_req.copy()
    snap.task_req[1, 2] = 0.5
    e = Engine()
    with pytest.raises(EngineError, match="fractional GPU"):
        e.load(snap)
    e.close()


def test_job_order_unit_cases_gpu():
    """The pop orders of actions/utils/job_order_by_queue_test.go (tests/test_job_order_units.py) on the engine: the
    visiting order of an allocate run where nothing fits, against the oracle and the reference's expected order."""
    import test_job_order_units as ju
    cases = [(c[1], c[2], c[3]) for c in ju.HIERARCHY]
    cases.append(({"test-queue": "test-parent", "test-parent": ""},
                  [("p150", 150, "test-queue"), ("p255", 255, "test-queue"), ("p160", 160, "test-queue"), ("p200", 200, "test-queue")],
                  ["p255", "p200", "p160", "p150"]))
    for queues, jobs, expected in cases:
        snap = ju.order_snapshot(queues, jobs)
        re_, ro = run_both(snap)
        assert_same(re_, ro)
        assert [jobs[int(j)][0] for j, _ in re_.visits] == expected


@pytest.mark.parametrize("k_value", [0.5, 2.0])
def test_historical_usage_and_k_value(k_value):
    """Time-based fair share inputs (SURVEY §8(f) rank 4): per-queue historical usage and the proportion plugin's kValue
    enter calcShareWeights (resource_division.go:224-251); over-subscribed queues so that the over-quota split decides
    who gets placed."""
    snap = synthetic.benchmark_snapshot(n_nodes=48, n_jobs=700, tasks_per_job=1, n_queues=8)
    rng = np.random.default_rng(11)
    Q = snap.n_queues
    snap.queue_usage = rng.choice(np.array([0.0, 0.05, 0.125, 0.25, 0.5]), size=(3, Q))
    snap.queue_deserved = snap.queue_deserved.copy()
    snap.queue_deserved[2, :8] = 16.0  # 8 leaf queues x 16 deserved GPUs < 384 GPUs: the rest is over-quota share
    cfg = abi.make_config(k_value=k_value)
    re_, ro = run_both(snap, cfg=cfg)
    assert_same(re_, ro)
    plain = Oracle(abi.make_config())
    snap2 = synthetic.benchmark_snapshot(n_nodes=48, n_jobs=700, tasks_per_job=1, n_queues=8)
    snap2.queue_deserved = snap.queue_deserved
    plain.load(snap2)
    assert not np.array_equal(plain.run("allocate").queue_fair_share, ro.queue_fair_share)  # usage is not vacuous


def test_tables_grid5_top_m_lists(monkeypatch):
    """Four scanners (not a power of two) with top-M lists on: the allocate and solver tables, a mixed 1 000-node
    snapshot and config4-small."""
    monkeypatch.setenv("KAI_GRID_EXACT", "5")
    for cid, case in ALLOCATE:
        snap, meta = dsl.build_snapshot(case["topology"])
        re_, ro = run_both(snap, cfg=case_config(case))
        assert_same(re_, ro)
    for cid, case in SOLVER:
        snap, meta = dsl.build_snapshot(case["topology"])
        re_, ro = run_both(snap, action=case["actions"][0])
        assert_same(re_, ro)
    snap = synthetic.benchmark_snapshot(n_nodes=1000, n_jobs=3000, tasks_per_job=2, n_queues=40, mixed=True)
    assert_same(*run_both(snap))
    snap = synthetic.config_snapshot("config4-small")
    assert_same(*run_both(snap))


@pytest.mark.parametrize("env", [("KAI_TRANSPORT", "persistent"), ("KAI_SEQUENCER", "device")])
def test_removed_modes_are_refused(env, monkeypatch):
    """The persistent transport and the device-resident sequencer no longer exist: selecting one fails the action
    with KAI_ERR_UNSUPPORTED and names the variable, instead of running the default path under the old name."""
    from kai_scheduler_b200.engine import EngineError
    snap = synthetic.benchmark_snapshot(n_nodes=16, n_jobs=20, tasks_per_job=1, n_queues=2)
    e = Engine()
    e.load(snap)
    monkeypatch.setenv(*env)
    with pytest.raises(EngineError, match=f"{env[0]}={env[1]}"):
        e.run("allocate")
    monkeypatch.delenv(env[0])
    assert_same(e.run("allocate"), run_both(snap)[1])
    e.close()


def test_300k_nodes_small_allocate():
    """300 000 nodes on one GPU: 256 scanners of ~1 172 rows, whose tiles fit k_record's shared memory.  A few hundred
    pods against the oracle."""
    snap = synthetic.benchmark_snapshot(n_nodes=300_000, n_jobs=300, tasks_per_job=2, n_queues=8, mixed=True)
    assert_same(*run_both(snap))


def test_resident_snapshot_reload_equals_full_load():
    """kai_snapshot.structure_epoch (ABI v7): a second load with the same epoch refreshes the per-cycle columns only (node
    idle / releasing / flags, task status / node, queue usage) and must behave exactly like a full load of the same data."""
    rng = np.random.default_rng(77)
    base = synthetic.reclaim_snapshot(n_nodes=96, running_per_node=6, victim_queues=3, reclaimer_jobs=24, reclaimer_tasks=2,
                                      reclaimer_gpus=3.0)
    e = Engine()
    base.structure_epoch = 41
    e.load(base)
    for act in ("allocate", "reclaim"):
        e.run(act)
    # next cycle: some running pods finished (their resources are free again), two nodes went NotReady
    nxt = synthetic.reclaim_snapshot(n_nodes=96, running_per_node=6, victim_queues=3, reclaimer_jobs=24, reclaimer_tasks=2,
                                     reclaimer_gpus=3.0)
    done = rng.choice(np.flatnonzero(nxt.task_status == abi.POD_RUNNING), size=60, replace=False)
    for t in done:
        nxt.node_idle[:, nxt.task_node[t]] += nxt.task_req[t]
    nxt.task_status[done] = abi.POD_STATUS_NAMES["Succeeded"]
    nxt.task_node[done] = -1
    nxt.node_flags[[5, 17]] &= ~np.uint32(abi.NODE_READY)
    nxt.structure_epoch = 41
    e.load(nxt)          # resident path
    full = Engine()
    nxt.structure_epoch = 0
    full.load(nxt)       # full path
    o = Oracle()
    o.load(nxt)
    for act in ("allocate", "consolidation", "reclaim", "preempt"):
        r1, r2, ro = e.run(act), full.run(act), o.run(act)
        assert_same(r1, ro)
        assert_same(r2, ro)
        assert r1.pods_evicted == ro.pods_evicted
    e.close()
    full.close()
    o.close()


def test_metric_cycle_small():
    """The allocate + reclaim cycle of bench.py's default configuration (synthetic.cycle_snapshot) at a size the oracle
    finishes in milliseconds; bench.py asserts the same at 50 000 nodes on every run."""
    snap = synthetic.config_snapshot("config3-cycle-small")
    e, o = Engine(), Oracle()
    e.load(snap)
    o.load(snap)
    evicted = 0
    for act in synthetic.CONFIG_ACTIONS["config3-cycle-small"]:
        re_, ro = e.run(act), o.run(act)
        assert_same(re_, ro)
        assert re_.pods_evicted == ro.pods_evicted
        evicted += re_.pods_evicted
    assert evicted == 16 and int((re_.task_status == abi.POD_PENDING).sum()) == 0
    e.close()
    o.close()
