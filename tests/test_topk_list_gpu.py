"""The idle-GPU filter's top-k list on over-committed GPU nodes (GPU box).

Reclaim and consolidation prune a scenario when the k rows with most idle + releasing GPUs cannot hold the pending
tasks.  On the GPU that list is k_record's per-scanner top-4 candidates, merged by k_merge_cluster and paged with a
cutoff until k rows are known.  Over-committed nodes (tests/value_regime.py, regime e) have negative keys, which the
merge must order below zero, and -0.0 keys, which equal +0.0 (the name rank decides).  Every run here is compared bit
for bit with the oracle, in the three modes of test_solver_host_sweep_gpu.py; "check" also compares every GPU and host
list with a plain restatement over all node rows, node by node.
"""
import re

import numpy as np
import pytest

import value_regime as vr
from kai_scheduler_b200 import abi, synthetic
from kai_scheduler_b200.engine import Engine
from oracle_lib import Oracle
from test_engine_gpu import assert_same
from test_solver_host_sweep_gpu import MODES

pytestmark = pytest.mark.gpu

E_REGIMES = [n for n in vr.REGIMES if n.startswith("e_")]
KNOBS = ("KAI_HOST_SWEEP_MAX", "KAI_HOST_SWEEP_CHECK", "KAI_GRID_EXACT", "KAI_PROFILE")


def _env(monkeypatch, mode, grid=None):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    if grid:
        monkeypatch.setenv("KAI_GRID_EXACT", grid)
    monkeypatch.setenv("KAI_PROFILE", "1")


def _topk_sweeps(err: str) -> int:
    """GPU top-k sweeps of the solver actions, from the KAI_PROFILE lines on stderr."""
    return sum(int(m) for m in re.findall(r"(\d+) top-k sweeps", err))


def _run(snap, cfg, action):
    actions = vr.ACTIONS if action == "cycle" else (action,)
    e, o = Engine(cfg), Oracle(cfg)
    e.load(snap)
    o.load(snap)
    for a in actions:
        re_, ro = e.run(a), o.run(a)
        assert_same(re_, ro)
        assert re_.pods_evicted == ro.pods_evicted, a
    e.close()
    o.close()


@pytest.mark.parametrize("action", ["reclaim", "consolidation", "cycle"])
@pytest.mark.parametrize("name", E_REGIMES)
@pytest.mark.parametrize("mode", sorted(MODES))
def test_topk_lists_match_oracle(mode, name, action, monkeypatch, capfd):
    _env(monkeypatch, mode)
    snap, cfg = vr.regime(name)
    _run(snap, cfg, action)
    sweeps = _topk_sweeps(capfd.readouterr().err)
    # the GPU merge answers lists in the gpu and check modes, and in the default mode once > 256 rows have free GPUs
    if action != "consolidation" and (mode != "default" or name == "e_overcommit_2048"):
        assert sweeps > 0


@pytest.mark.parametrize("grid", ["2", "5"])
@pytest.mark.parametrize("name", E_REGIMES)
def test_topk_lists_on_forced_grids(name, grid, monkeypatch, capfd):
    """One scanner (KAI_GRID_EXACT=2) or four (=5), every list on the GPU: the pages cross from keys >= 0 into negative
    ones, and a scanner's 4th candidate is negative while it has more rows."""
    _env(monkeypatch, "gpu", grid)
    snap, cfg = vr.regime(name)
    if grid == "2" and snap.n_nodes >= 2048:
        pytest.skip("one scanner cannot hold 2048 node rows (test_value_regime_gpu.test_regime_paths covers the refusal)")
    _run(snap, cfg, "cycle")
    assert _topk_sweeps(capfd.readouterr().err) > 0


def _signed_zero_snapshot():
    """32 full nodes (8 running 1-GPU pods each) whose Idle and Releasing GPUs are -0.0 on every other name rank and
    +0.0 on the rest, and one pending 4 x 8-GPU gang: reclaim's filter lists the 4 rows with most idle GPUs, all zero,
    which must be the 4 lowest name ranks whatever the sign of their zero."""
    snap = synthetic.reclaim_snapshot(32, victim_queues=2, reclaimer_jobs=1, reclaimer_tasks=4, reclaimer_gpus=8.0)
    G = abi.RES_GPU
    assert (snap.node_idle[G] == 0).all()
    minus = (snap.node_name_rank % 2) == 1
    snap.node_idle[G, minus] = -0.0
    snap.node_releasing[G, minus] = -0.0
    return snap


def test_signed_zero_rows_list_by_name_rank(monkeypatch, capfd):
    _env(monkeypatch, "check")
    snap = _signed_zero_snapshot()
    assert np.signbit(snap.node_idle[abi.RES_GPU]).sum() == 16
    _run(snap, abi.make_config(), "reclaim")
    assert _topk_sweeps(capfd.readouterr().err) > 0

