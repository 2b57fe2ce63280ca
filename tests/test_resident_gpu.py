"""The resident snapshot (kai_snapshot.structure_epoch, ABI v7) over many cycles on the GPU.

A long-lived engine that reloads the same structure every cycle refreshes only the per-cycle columns
(include/kai_engine.h).  Every test here runs cycles through that path and compares each action with a fresh engine
that loads the same snapshot in full (epoch 0) and with the CPU oracle, bit for bit.  The cycles come from
tests/resident_lib.next_cycle: the outcome of a cycle written back as the reference's integration harness does, plus
random status-only events.  KAI_RESIDENT_CHECK=1 is set throughout, so a resident load of a snapshot whose structure
changed fails loudly instead of running on stale tables.
"""
import time

import numpy as np
import pytest

import dsl
import resident_lib as rl
from fixtures import action_cases
from kai_scheduler_b200 import abi, synthetic
from kai_scheduler_b200.engine import Engine, EngineError
from oracle_lib import Oracle
from test_engine_gpu import assert_same
from test_snapshot_io import _random_topology

pytestmark = pytest.mark.gpu

ACTIONS = ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"]
FUZZ_CFG = dict(allow_consolidating_reclaim=True, max_consolidation_preemptees=-1, staleness_grace_period_s=60)
INTEGRATION = action_cases(["integration_tests__"])


@pytest.fixture(autouse=True)
def resident_check(monkeypatch):
    monkeypatch.setenv("KAI_RESIDENT_CHECK", "1")


def three_way(rr, snap, actions, cfg=None, what=""):
    """Load `snap` on the resident runner, a fresh engine (full load) and the oracle; run `actions` on all three and
    compare every result.  Returns the resident engine's results."""
    full, o = Engine(cfg), Oracle(cfg)
    rr.load(snap)
    full.load(rl.full_load_copy(snap))
    o.load(snap)
    out = []
    try:
        for act in actions:
            r1, r2, ro = rr.run(act), full.run(act), o.run(act)
            try:
                assert_same(r2, ro)
                assert r2.pods_evicted == ro.pods_evicted
                assert_same(r1, ro)
                assert r1.pods_evicted == ro.pods_evicted
            except AssertionError as ex:
                raise AssertionError(f"{what} action {act}: {ex}") from None
            out.append(ro)
    finally:
        full.close()
        o.close()
    return out


def run_cycles(snap, rng, cfg, cycles=5, actions=ACTIONS, what="", full_every=0):
    """`cycles` cycles of `snap` on one resident engine; returns the runner's (loads, resident loads)."""
    rr = rl.ResidentRunner(lambda: Engine(cfg))
    try:
        for c in range(cycles):
            if full_every and c and c % full_every == 0:
                rr.force_full()
            res = three_way(rr, snap, actions, cfg, what=f"{what} cycle {c}")
            snap = rl.next_cycle(snap, res[-1], rng)
        return rr.loads, rr.resident_loads
    finally:
        rr.close()


# ---------------------------------------------------------------- integration tables on one resident engine

def test_integration_tables_on_one_resident_engine():
    """All 60 multi-round integration tables; each table's rounds share one engine, so every round after the first
    reloads resident.  The reference's expectations hold and every round's state after every action equals the
    oracle's (as in test_engine_gpu.test_integration_tables_gpu)."""
    import copy
    t0 = time.time()
    loads = resident = 0
    for cid, case in INTEGRATION:
        e_case, o_case = copy.deepcopy(case), copy.deepcopy(case)
        seen = {"e": [], "o": []}
        shared = rl.ResidentRunner(Engine)

        class Tap:
            def __init__(self, inner, key):
                self.inner, self.key = inner, key

            def load(self, snap):
                self.inner.load(snap)

            def run(self, action):
                r = self.inner.run(action)
                seen[self.key].append((r.task_status.copy(), r.task_node.copy(), r.node_idle.copy(), r.node_releasing.copy(),
                                       r.queue_allocated.copy(), r.visits.copy()))
                return r

            def close(self):  # the engine outlives the round
                pass

        errs = dsl.run_integration_case(e_case, lambda: Tap(shared, "e"))
        assert not errs, f"{case['source']} #{case['index']}: {errs[:3]}"
        dsl.run_integration_case(o_case, lambda: Tap(Oracle(), "o"))
        assert len(seen["e"]) == len(seen["o"])
        for k, (a, b) in enumerate(zip(seen["e"], seen["o"])):
            for x, y in zip(a, b):
                np.testing.assert_array_equal(x, y, err_msg=f"{cid} step {k}")
        loads += shared.loads
        resident += shared.resident_loads
        shared.close()
    print(f"\nintegration tables: {loads} rounds, {resident} resident, {time.time() - t0:.1f} s")
    # tests/test_resident_sim.py: the rebuilt structure never changes between rounds
    assert resident == loads - len(INTEGRATION) and resident >= 360


# ---------------------------------------------------------------- multi-cycle fuzz

@pytest.mark.parametrize("chunk", range(8))
def test_resident_cycles_random_clusters(chunk):
    t0 = time.time()
    loads = resident = 0
    for seed in range(chunk * 25, (chunk + 1) * 25):
        rng = np.random.default_rng(9000 + seed)
        snap = rl.prepare(dsl.build_snapshot(_random_topology(rng))[0], rng)
        a, b = run_cycles(snap, rng, abi.make_config(**FUZZ_CFG), what=f"seed {seed}")
        loads, resident = loads + a, resident + b
    print(f"\nchunk {chunk}: {loads} cycles, {resident} resident, {time.time() - t0:.1f} s")
    assert resident == loads - 25


SYNTHETIC = [
    ("reclaim", dict(n_nodes=48, running_per_node=7, victim_queues=2, reclaimer_jobs=12, reclaimer_tasks=2, reclaimer_gpus=3.0)),
    ("reclaim", dict(n_nodes=96, running_per_node=6, victim_queues=4, reclaimer_jobs=24, reclaimer_tasks=2, reclaimer_gpus=3.0)),
    ("reclaim", dict(n_nodes=24, running_per_node=6, victim_queues=3, reclaimer_jobs=20, reclaimer_tasks=3, reclaimer_gpus=3.0)),
    ("topology", dict(n_nodes=300, n_gangs=50, nodes_per_rack=5, racks_per_leaf=3, leaves_per_spine=2, running_fraction=0.5, max_pods=6)),
    ("topology", dict(n_nodes=96, n_gangs=20, nodes_per_rack=4, racks_per_leaf=3, leaves_per_spine=2, running_fraction=0.6, max_pods=4)),
]


@pytest.mark.parametrize("kind,kw", SYNTHETIC, ids=[f"{k}-n{kw['n_nodes']}" for k, kw in SYNTHETIC])
def test_resident_cycles_synthetic(kind, kw):
    rng = np.random.default_rng(kw["n_nodes"])
    snap = synthetic.reclaim_snapshot(**kw) if kind == "reclaim" else synthetic.topology_snapshot(**kw)
    loads, resident = run_cycles(rl.prepare(snap, rng), rng, abi.make_config(**FUZZ_CFG), what=kind)
    assert resident == loads - 1


PATHS = [
    ("grid2", {"KAI_GRID_EXACT": "2"}, ACTIONS),
    ("grid5", {"KAI_GRID_EXACT": "5"}, ACTIONS),
    ("no-topm", {"KAI_NO_TOPM": "1"}, ACTIONS),
]


@pytest.mark.parametrize("name,env,actions", PATHS, ids=[p[0] for p in PATHS])
def test_resident_cycles_every_path(monkeypatch, name, env, actions):
    """The fuzz subset through forced grids and single-candidate answers."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for seed in range(30):
        rng = np.random.default_rng(9000 + seed)
        snap = rl.prepare(dsl.build_snapshot(_random_topology(rng))[0], rng)
        run_cycles(snap, rng, abi.make_config(**FUZZ_CFG), cycles=4, actions=actions, what=f"{name} seed {seed}")


# ---------------------------------------------------------------- targeted regressions

def _small_cluster(n_nodes=3, gpus=4, jobs=(("queue0", 1, 1),), queues=("queue0",)):
    topo = {"Nodes": {f"node{i}": {"GPUs": gpus} for i in range(n_nodes)},
            "Queues": [{"Name": q, "DeservedGPUs": 1} for q in queues],
            "Jobs": [{"Name": f"job{k}", "QueueName": q, "Priority": 100, "RequiredGPUsPerTask": g,
                      "Tasks": [{"State": "Pending"} for _ in range(n)]} for k, (q, n, g) in enumerate(jobs)]}
    return rl.prepare(dsl.build_snapshot(topo)[0])


def _bindings(snap, actions, cfg=None):
    o = Oracle(cfg)
    o.load(snap)
    res = [o.run(a) for a in actions][-1]
    o.close()
    return res


def _two_cycles(a, b, actions, cfg=None):
    """Cycle a, then cycle b under the same epoch on one engine; each compared with a full load and the oracle."""
    rr = rl.ResidentRunner(lambda: Engine(cfg))
    try:
        three_way(rr, a, actions, cfg, what="first cycle")
        three_way(rr, b, actions, cfg, what="second cycle")
        assert (rr.loads, rr.resident_loads) == (2, 1)
    finally:
        rr.close()


def nominated_pair():
    a = _small_cluster()
    b = rl.next_cycle(a, a, None, events=())
    a.task_nominated[0] = 2
    b.task_nominated[0] = 1
    return a, b


def test_nominated_node_moves_under_the_same_epoch():
    """Status.NominatedNodeName is a pod status field: it changes without an epoch bump and must be re-read."""
    a, b = nominated_pair()
    assert _bindings(a, ["allocate"]).task_node[0] == 2 and _bindings(b, ["allocate"]).task_node[0] == 1
    _two_cycles(a, b, ["allocate"])


def foreign_pair():
    a = _small_cluster()
    b = rl.next_cycle(a, a, None, events=())
    b.node_foreign[:, 1] = [4000.0, 4e9, 2.0]
    b.node_idle[:3, 1] -= b.node_foreign[:, 1]
    return a, b


def test_foreign_pods_change_under_the_same_epoch():
    """Pods of other schedulers start: the fair-share totals (proportion.go:276-286) shrink."""
    a, b = foreign_pair()
    assert not np.array_equal(_bindings(a, ["allocate"]).total_resource, _bindings(b, ["allocate"]).total_resource)
    _two_cycles(a, b, ["allocate"])


def usage_pair():
    topo = {"Nodes": {"node0": {"GPUs": 1}},
            "Queues": [{"Name": q, "DeservedGPUs": 0, "GPUOverQuotaWeight": 1} for q in ("queue0", "queue1")],
            "Jobs": [{"Name": f"job{k}", "QueueName": q, "Priority": 100, "RequiredGPUsPerTask": 1, "Tasks": [{"State": "Pending"}]}
                     for k, q in enumerate(("queue0", "queue1"))]}
    a = rl.prepare(dsl.build_snapshot(topo)[0])
    b = rl.next_cycle(a, a, None, events=())
    a.queue_usage[:, 0] = 0.75
    b.queue_usage[:, 1] = 0.75
    return a, b


def test_queue_usage_reorders_queues_under_the_same_epoch():
    """Historical usage moves the over-quota fair share from one queue to the other: the queues swap places."""
    a, b = usage_pair()
    ra, rb = _bindings(a, ["allocate"]), _bindings(b, ["allocate"])
    assert ra.visits[0, 0] != rb.visits[0, 0], "the usage drift no longer reorders the queues"
    _two_cycles(a, b, ["allocate"])


def min_runtime_pair():
    a = synthetic.reclaim_snapshot(n_nodes=8, running_per_node=6, victim_queues=3, reclaimer_jobs=4, reclaimer_tasks=2,
                                   reclaimer_gpus=3.0)
    a = rl.prepare(a, min_runtimes=False)
    a.queue_reclaim_min_runtime_s = np.full(a.n_queues, 300.0)
    a.job_last_start_s[a.job_last_start_s > 0] = a.now_s - 100.0
    b = rl.next_cycle(a, a, None, events=())
    b.now_s = a.now_s + 400.0
    return a, b


def test_now_crosses_a_min_runtime_under_the_same_epoch():
    a, b = min_runtime_pair()
    assert _bindings(a, ["reclaim"]).pods_evicted == 0 and _bindings(b, ["reclaim"]).pods_evicted > 0
    _two_cycles(a, b, ["allocate", "reclaim"])


STALE_CFG = dict(staleness_grace_period_s=60)


def stale_pair():
    topo = {"Nodes": {"node0": {"GPUs": 1}}, "Queues": [{"Name": "queue0", "DeservedGPUs": 1}],
            "Jobs": [{"Name": "job0", "QueueName": "queue0", "Priority": 100, "RequiredGPUsPerTask": 1,
                      "Tasks": [{"State": "Running", "NodeName": "node0"}, {"State": "Pending"}]}]}
    a = rl.prepare(dsl.build_snapshot(topo)[0])
    a.job_stale_since_s[0] = a.now_s - 10.0
    b = rl.next_cycle(a, a, None, events=())
    b.now_s = a.now_s + 100.0
    return a, b


def test_stale_stamp_expires_under_the_same_epoch():
    a, b = stale_pair()
    cfg = abi.make_config(**STALE_CFG)
    assert _bindings(a, ACTIONS, cfg).pods_evicted == 0 and _bindings(b, ACTIONS, cfg).pods_evicted > 0
    _two_cycles(a, b, ACTIONS, cfg)


def not_ready_pair():
    a = _small_cluster()
    b = rl.next_cycle(a, a, None, events=())
    b.node_flags[2] &= ~np.uint32(abi.NODE_READY)
    return a, b


def test_node_goes_not_ready_under_the_same_epoch():
    a, b = not_ready_pair()
    assert not np.array_equal(_bindings(a, ["allocate"]).total_resource, _bindings(b, ["allocate"]).total_resource)
    _two_cycles(a, b, ["allocate"])


def test_shape_change_under_the_same_epoch_loads_in_full():
    """An optional array that appears changes the engine's shape key: a full load although the epoch is unchanged."""
    a, b = nominated_pair()
    a.task_nominated = None
    assert _bindings(a, ["allocate"]).task_node[0] != _bindings(b, ["allocate"]).task_node[0]
    e, o = Engine(), Oracle()
    try:
        for snap in (a, b):
            snap.structure_epoch = 41
            e.load(snap)
            o.load(snap)
            assert_same(e.run("allocate"), o.run("allocate"))
    finally:
        e.close()
        o.close()


def test_epoch_zero_always_loads_in_full():
    """Epoch 0 is never resident: a structural edit between two epoch-0 loads is used, not refused."""
    a = _small_cluster(jobs=(("queue0", 1, 1),))
    b = rl.full_load_copy(a)
    b.task_req = a.task_req.copy()
    b.task_req[0, abi.RES_GPU] = 8.0  # no longer fits on any node
    assert _bindings(a, ["allocate"]).task_node[0] >= 0 and _bindings(b, ["allocate"]).task_node[0] < 0
    e, o = Engine(), Oracle()
    try:
        for snap in (a, b, a):
            snap.structure_epoch = 0
            e.load(snap)
            o.load(snap)
            assert_same(e.run("allocate"), o.run("allocate"))
    finally:
        e.close()
        o.close()


# ---------------------------------------------------------------- contract check

def every_structural_field_snapshot():
    """A topology cluster with every optional structural array present (and valid)."""
    rng = np.random.default_rng(11)
    s = synthetic.topology_snapshot(n_nodes=64, n_gangs=10, nodes_per_rack=4, racks_per_leaf=2, leaves_per_spine=2,
                                    running_fraction=0.3, max_pods=4)
    s = rl.prepare(s, rng)
    J, S, N, T = s.n_jobs, s.n_podsets, s.n_nodes, s.n_tasks
    s.node_gpu_count = s.node_allocatable[abi.RES_GPU].copy()
    s.pred_mask = np.full((2, (N + 31) // 32), 0xffffffff, dtype=np.uint32)
    s.pred_mask[1, 0] = 0xfffffff0
    s.task_pred_class = (np.arange(T) % 3 - 1).astype(np.int32)
    s.job_signature = (np.arange(J) % 4).astype(np.int32)
    ps_job = np.repeat(np.arange(J), np.diff(s.job_podset_begin)).astype(np.int32)
    s.job_sgs_begin = np.arange(J + 1, dtype=np.int32)
    s.sgs_parent = np.full(J, -1, dtype=np.int32)
    s.sgs_name_rank = np.zeros(J, dtype=np.int32)
    s.sgs_topology = s.job_topology.copy()
    s.sgs_required_level = s.job_required_level.copy()
    s.sgs_preferred_level = s.job_preferred_level.copy()
    s.podset_sgs = ps_job
    s.podset_topology = np.full(S, -1, dtype=np.int32)
    s.podset_required_level = np.full(S, -1, dtype=np.int32)
    s.podset_preferred_level = np.full(S, -1, dtype=np.int32)
    missing = [n for n in rl.STRUCTURAL_FIELDS if getattr(s, n) is None]
    assert not missing, missing
    return s


def test_structural_edit_under_the_same_epoch_is_refused():
    base = every_structural_field_snapshot()
    base.structure_epoch = 41
    e, o = Engine(), Oracle()
    o.load(base)
    e.load(base)
    assert_same(e.run("allocate"), o.run("allocate"))
    o.close()
    checked = []
    try:
        for name in rl.STRUCTURAL_FIELDS:
            if name == "n_res":  # part of the shape key: a change is a full load by itself
                continue
            e.load(base)  # a full load after the refused one below, or resident with an unchanged structure
            edited = rl.full_load_copy(base)
            arr = np.array(getattr(base, name), copy=True)
            flat = arr.reshape(-1)
            flat[0] = flat[0] + 1
            setattr(edited, name, arr)
            edited.structure_epoch = 41
            with pytest.raises(EngineError, match=f"{name} changed under structure_epoch 41"):
                e.load(edited)
            checked.append(name)
        # an unchanged structure under the same epoch still loads resident (no false alarm)
        e.load(base)
        nxt = rl.next_cycle(base, base, np.random.default_rng(5))
        nxt.structure_epoch = 41
        e.load(nxt)
    finally:
        e.close()
    assert len(checked) == len(rl.STRUCTURAL_FIELDS) - 1
