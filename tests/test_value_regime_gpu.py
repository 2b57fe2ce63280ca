"""Engine == oracle, bit for bit, on non-round resource values (tests/value_regime.py; GPU box only).

Every regime runs allocate, consolidation, reclaim, preempt and stalegangeviction on one session and compares every
table of every action with the oracle, the fair shares included (k_fair_share uses the oracle's operations: no
tolerance).  The same runs repeat on two fresh engines and a resident reload (the bits must not change from run to
run), under forced grids, with single-candidate answers and without the fresh-gang bulk path.  test_value_regime.py shows on the CPU that each regime reaches the case it targets.
"""
import functools

import numpy as np
import pytest

import value_regime as vr
from kai_scheduler_b200.engine import Engine, EngineError
from oracle_lib import Oracle
from test_engine_gpu import assert_same

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _oracle_cycle(name, actions=vr.ACTIONS):
    snap, cfg = vr.regime(name)
    o = Oracle(cfg)
    o.load(snap)
    out = [o.run(a) for a in actions]
    o.close()
    return out


def _engine_cycle(eng, snap, actions=vr.ACTIONS):
    eng.load(snap)
    return [eng.run(a) for a in actions]


def _check(res_e, res_o):
    for a, re_, ro in zip(vr.ACTIONS, res_e, res_o):
        assert_same(re_, ro)
        np.testing.assert_array_equal(re_.queue_fair_share, ro.queue_fair_share, err_msg=a)
        assert re_.pods_evicted == ro.pods_evicted, a


@pytest.mark.parametrize("name", vr.REGIMES)
def test_regime_cycle_matches_oracle(name):
    snap, cfg = vr.regime(name)
    e = Engine(cfg)
    _check(_engine_cycle(e, snap), _oracle_cycle(name))
    e.close()


@pytest.mark.parametrize("name", vr.REGIMES)
def test_regime_runs_are_deterministic(name):
    """Two fresh engines and a resident reload of the first give the same bits (atomics are unordered run to run)."""
    snap, cfg = vr.regime(name)
    snap.structure_epoch = 5
    e1, e2 = Engine(cfg), Engine(cfg)
    r1 = _engine_cycle(e1, snap)
    r2 = _engine_cycle(e2, snap)
    r3 = _engine_cycle(e1, snap)      # same epoch: the resident path
    for a, b in ((r1, r2), (r1, r3)):
        _check(a, b)
    _check(r1, _oracle_cycle(name))
    e1.close()
    e2.close()


KNOBS = [("KAI_GRID_EXACT", "2"), ("KAI_GRID_EXACT", "5"), ("KAI_NO_TOPM", "1"), ("KAI_NO_GANG_FAST", "1")]


@pytest.mark.parametrize("knob", KNOBS, ids=[f"{k}={v}" for k, v in KNOBS])
@pytest.mark.parametrize("name", vr.REGIMES)
def test_regime_paths(name, knob, monkeypatch):
    monkeypatch.setenv(*knob)
    snap, cfg = vr.regime(name)
    e = Engine(cfg)
    if knob == ("KAI_GRID_EXACT", "2") and snap.n_nodes >= 2048:
        # one scanner CTA would have to hold every node row in shared memory (100 B a row with 4 resources, 227 KB of
        # shared memory per CTA on an H100, 40 KB of it kept for k_record): the engine refuses instead of guessing
        with pytest.raises(EngineError, match="node tile does not fit"):
            e.load(snap)
        e.close()
        return
    _check(_engine_cycle(e, snap), _oracle_cycle(name))
    e.close()


@pytest.mark.parametrize("name", ["a_totals", "b_queues", "d_shares"])
def test_open_session_tables_are_the_ordered_sums(name):
    """No pending pod: total_resource and the queue tables come straight from k_node_totals / k_queue_usage.  They equal
    the oracle's bits, and the exact sum within the sequential rounding bound."""
    snap, cfg = vr.regime(name)
    snap = vr.without_pending(snap)
    e, o = Engine(cfg), Oracle(cfg)
    e.load(snap)
    o.load(snap)
    re_, ro = e.fair_share(), o.fair_share()
    e.close()
    o.close()
    for field in ("total_resource", "queue_request", "queue_allocated", "queue_allocated_non_preemptible",
                  "queue_fair_share"):
        np.testing.assert_array_equal(getattr(re_, field), getattr(ro, field), err_msg=field)
    for r in range(3):
        v = vr.node_summands(snap, r)
        assert abs(vr.exact([re_.total_resource[r]]) - vr.exact(v)) <= vr.sequential_bound(v)
    for q in range(snap.n_queues):
        for field, table in (("request", re_.queue_request), ("allocated", re_.queue_allocated),
                             ("allocated_np", re_.queue_allocated_non_preemptible)):
            v = vr.queue_summands(snap, q, 1, field)
            assert abs(vr.exact([table[1, q]]) - vr.exact(v)) <= vr.sequential_bound(v), (q, field)
