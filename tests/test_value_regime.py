"""The value regimes of tests/value_regime.py reach the cases they target (CPU only).

These checks are what make test_value_regime_gpu.py meaningful: on round inputs every order of summation and every
equal form of a score give the same bits, so engine == oracle proves nothing about order or association.
"""
from fractions import Fraction

import numpy as np
import pytest

import value_regime as vr
from kai_scheduler_b200 import abi
from oracle_lib import Oracle, lib


def _open_session(snap, cfg=None):
    o = Oracle(cfg)
    o.load(snap)
    res = o.fair_share()
    o.close()
    return res


@pytest.mark.parametrize("name", ["a_totals", "a_totals_1800"])
def test_a_node_memory_total_is_inexact_and_order_dependent(name):
    snap, _ = vr.regime(name)
    assert snap.n_nodes >= (5000 if name == "a_totals" else 1800)
    M = abi.RES_MEM
    v = vr.node_summands(snap, M)
    assert (v == np.floor(v)).all() and (v % 2 == 1).all()  # odd byte counts: granularity 1 B
    ex = vr.exact(v)
    assert ex > 2 ** 53
    tot = _open_session(snap).total_resource[M]
    assert tot == vr.sequential(v)                   # the oracle adds in ascending node index
    assert Fraction(tot) != ex
    assert abs(Fraction(tot) - ex) <= vr.sequential_bound(v)
    assert vr.kernel_order_total(snap, M) != tot     # k_node_totals' tree order, blocks' atomics in index order
    rng = np.random.default_rng(0)
    blocks = min(vr.H100_SMS * 4, (snap.n_nodes + 255) // 256)
    assert any(vr.kernel_order_total(snap, M, block_order=rng.permutation(blocks)) != tot for _ in range(8))
    # the node CPU values are arbitrary milli values, not round thousands
    assert (snap.node_allocatable[0] % 1000 != 0).mean() > 0.9


def test_b_queue_sums_are_inexact_and_order_dependent():
    snap = vr.inexact_queue_sums()
    assert snap.n_tasks >= 10_000
    assert ((snap.task_status == abi.POD_RUNNING).sum() > 0) and ((snap.task_status == abi.POD_PENDING).sum() > 0)
    pre = (snap.job_flags & abi.JOB_PREEMPTIBLE) != 0
    assert pre.any() and (~pre).any()
    assert len(set(snap.queue_parent[snap.queue_parent >= 0].tolist())) == 1  # one department above the leaf queues
    res = _open_session(snap)
    dept = int(np.flatnonzero(snap.queue_parent < 0)[0])
    tables = {"request": res.queue_request, "allocated": res.queue_allocated,
              "allocated_np": res.queue_allocated_non_preemptible}
    for field, table in tables.items():
        v = vr.queue_summands(snap, dept, abi.RES_MEM, field)
        got = table[abi.RES_MEM, dept]
        ex = vr.exact(v)
        assert ex > 2 ** 53, field
        assert got == vr.sequential(v), field          # job, podset, task order
        assert Fraction(got) != ex, field
        assert abs(Fraction(got) - ex) <= vr.sequential_bound(v), field
        assert got != vr.sequential(v[::-1]) or got != vr.pairwise(v), field


@pytest.mark.parametrize("wide", [2.0 ** 47, 2.0 ** 49])
def test_c_binpack_winners_beat_the_runner_up_by_a_few_ulps(wide):
    """Every sweep of the oracle's allocate, replayed with its own binpack score: the replay picks the oracle's node each
    time, some winners beat the runner-up by 1 to 8 ulps, and some tie with it exactly (the name rank decides)."""
    snap = vr.score_near_ties(wide=wide)
    o = Oracle()
    o.load(snap)
    res = o.run("allocate")
    o.close()
    gaps, mismatches = vr.binpack_sweeps(snap, res)
    assert len(gaps) == snap.n_tasks and mismatches == 0
    assert ((gaps > 0) & (gaps <= 8)).any()
    assert (gaps == 0).any()
    # an algebraically equal form of pack.go:45-64 gives other bits on some node of the first sweep
    cur = snap.node_idle[abi.RES_CPU] + snap.node_releasing[abi.RES_CPU]
    A = snap.node_allocatable[abi.RES_CPU]
    mn, mx = cur[A != 0].min(), cur[A != 0].max()
    f = lib().kai_oracle_binpack_score
    ref = np.array([f(mn, mx, c, a) for c, a in zip(cur, A)])
    assert (9.0 * (mx - cur) / (mx - mn) != ref).any()


def test_c_edges_reach_every_branch_of_the_binpack_score():
    snap = vr.score_edges()
    A, cur = snap.node_allocatable[0], snap.node_idle[0] + snap.node_releasing[0]
    assert (A == 0).any()                                        # overall == 0
    cpu_only = snap.node_allocatable[2] == 0
    nz = cpu_only & (A != 0)
    assert nz.any() and cur[nz].min() == cur[nz].max()           # mn == mx among the CPU-only nodes with CPU
    assert (snap.task_req[:, 0] == 0).any() and (snap.task_req[:, 2] == 0).any()
    f = lib().kai_oracle_binpack_score
    assert f(5.0, 5.0, 5.0, 1.0) == 9.0 and f(0.0, 0.0, 0.0, 1.0) == 0.0 and f(1.0, 3.0, 2.0, 0.0) == 0.0


def test_d_fair_shares_take_the_fractional_paths():
    snap, k = vr.fractional_shares()
    assert k != int(k)
    assert (snap.queue_usage != np.round(snap.queue_usage)).any()
    assert (snap.queue_oqw != np.round(snap.queue_oqw)).any()
    res = _open_session(snap, abi.make_config(k_value=k))
    assert (res.total_resource[0] != np.floor(res.total_resource[0]))          # a non-integer CPU total
    fair = res.queue_fair_share
    assert (fair != np.floor(fair)).any()
    mine, paths = vr.fair_share_paths(snap, k, res)
    np.testing.assert_array_equal(mine, fair)   # the restatement follows the oracle bit for bit ...
    assert paths["floor_with_remainder"] > 0    # ... and took floor(fs) with a remainder left over
    assert paths["fractional_remainder_gift"] > 0  # and fmin(1.0, remaining) with a fractional remaining


def test_regimes_keep_node_accounting_consistent():
    """Idle + the placed pods' requests (Pipelined ones aside) + the foreign pods = Allocatable on every node, and
    Releasing = the Releasing pods' requests - the Pipelined pods' requests.  Only the over-committed regimes (e) have
    nodes with negative Idle."""
    for name in vr.REGIMES:
        snap, _ = vr.regime(name)
        used = np.zeros_like(snap.node_allocatable)
        rel = np.zeros_like(snap.node_allocatable)
        for t in np.flatnonzero(snap.task_node >= 0):
            n, st = snap.task_node[t], snap.task_status[t]
            if st == abi.POD_PIPELINED:
                rel[:, n] -= snap.task_req[t]
                continue
            used[:, n] += snap.task_req[t]
            if st == abi.POD_RELEASING:
                rel[:, n] += snap.task_req[t]
        if snap.node_foreign is not None:
            used[:3] += snap.node_foreign
        np.testing.assert_array_equal(snap.node_idle + used - snap.node_allocatable, 0, err_msg=name)
        np.testing.assert_array_equal(snap.node_releasing - rel, 0, err_msg=name)
        if not name.startswith("e_"):
            assert (snap.node_idle[:3] >= 0).all(), name


E_REGIMES = [n for n in vr.REGIMES if n.startswith("e_")]


@pytest.mark.parametrize("name", E_REGIMES)
def test_e_overcommitted_rows_reach_the_negative_list_keys(name):
    """The over-committed regimes put negative idle-GPU keys where the top-k list's sort and cut meet them."""
    snap, cfg = vr.regime(name)
    G, N = abi.RES_GPU, snap.n_nodes
    idle, rel, alloc = snap.node_idle[G], snap.node_releasing[G], snap.node_allocatable[G]
    key = vr.idle_gpu_key(snap)
    assert (idle < 0).sum() >= N // 4 and set(np.unique(idle[(idle < 0) & (alloc > 0)])) >= {-1.0, -2.0, -3.0}
    assert ((idle < 0) & (rel > 0)).any()                       # Releasing pod on an over-committed node
    assert (rel < 0).any()                                      # Pipelined pod
    assert ((alloc == 0) & (idle < 0)).sum() == 2               # binpack's overall == 0 skip with pods running
    assert ((alloc != 0) & (idle < 0)).any()                    # binpack's minimum is negative
    mz = (key == 0) & np.signbit(key)
    assert mz.sum() >= 3 and np.signbit(idle[mz]).all() and np.signbit(rel[mz]).all()
    pz = np.flatnonzero((key == 0) & ~np.signbit(key))
    assert len(pz) > 0 and snap.node_name_rank[pz].min() < snap.node_name_rank[mz].max()   # -0.0 and +0.0 ranks interleave
    # the page-and-cut loop meets a negative cut: with 4 scanners (KAI_GRID_EXACT=5) and, where a scanner of the default
    # grid (min(256, N) scanners) holds >= 5 rows, there too
    assert vr.stripe_cut_goes_negative(snap, 4)
    if N // min(256, N) >= 5:
        assert vr.stripe_cut_goes_negative(snap, min(256, N))
    # the filter needs more rows than have a key >= 0 (e_overcommit), or more than 256 rows have free GPUs, which is
    # past the host answer's default limit (e_overcommit_2048)
    gangs = np.diff(snap.podset_task_begin)[snap.task_status[snap.podset_task_begin[:-1]] == abi.POD_PENDING]
    if name == "e_overcommit":
        assert gangs.max() > (key >= 0).sum()
    else:
        assert (key > 0).sum() > 256


@pytest.mark.parametrize("name,action", [("e_overcommit", "reclaim"), ("e_overcommit_2048", "consolidation"),
                                         ("e_overcommit_2048", "reclaim")])
def test_e_workloads_evict(name, action):
    """The oracle's reclaim and consolidation evict pods on these clusters: the engine's victims are compared, not an
    empty answer."""
    snap, cfg = vr.regime(name)
    o = Oracle(cfg)
    o.load(snap)
    res = o.run(action)
    o.close()
    assert res.pods_evicted > 0
