"""Restricted simulation sweeps answered on the host (GPU box).

The solver answers a simulation sweep whose feasible-node set holds at most KAI_HOST_SWEEP_MAX rows, and the idle-GPU
filter's top-k list when the rows it needs are known from the mirror, from its node mirror instead of a GPU round trip.  Every solver workload of the GPU suite runs here three ways, each bit for bit
against the oracle:
  * "default":  the default maximum (small sets on the host, the rest on the GPU);
  * "gpu":      KAI_HOST_SWEEP_MAX=0, every sweep on the GPU (the path before host answers existed);
  * "gpu-split": as "gpu", with KAI_NO_FUSED_LAUNCH=1: a sweep's binpack extremes come from a MINMAX launch followed by
                the sweep launch instead of the exchange inside one cooperative launch;
  * "check":    every eligible sweep and top-k list answered on the host AND on the GPU (KAI_HOST_SWEEP_CHECK=1),
                the action fails on any difference (node, score bits, name rank, flags; the listed rows).
"""
import pytest

import test_cycle_fuzz_gpu as cycle_fuzz
import test_engine_gpu as engine_gpu
import test_value_regime_gpu as regime_gpu
import value_regime as vr
from kai_scheduler_b200 import synthetic
from kai_scheduler_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODES = {
    "default": {},
    "gpu": {"KAI_HOST_SWEEP_MAX": "0"},
    "gpu-split": {"KAI_HOST_SWEEP_MAX": "0", "KAI_NO_FUSED_LAUNCH": "1"},
    "check": {"KAI_HOST_SWEEP_MAX": "100000000", "KAI_HOST_SWEEP_CHECK": "1"},
}


@pytest.fixture(params=sorted(MODES))
def sweep_mode(request, monkeypatch):
    monkeypatch.delenv("KAI_HOST_SWEEP_MAX", raising=False)
    monkeypatch.delenv("KAI_HOST_SWEEP_CHECK", raising=False)
    monkeypatch.delenv("KAI_NO_FUSED_LAUNCH", raising=False)
    for k, v in MODES[request.param].items():
        monkeypatch.setenv(k, v)
    return request.param


@pytest.mark.parametrize("cid,case", engine_gpu.SOLVER, ids=[c[0] for c in engine_gpu.SOLVER])
def test_solver_tables(sweep_mode, cid, case):
    engine_gpu.test_solver_tables_gpu(cid, case)


@pytest.mark.parametrize("cid,case", engine_gpu.INTEGRATION, ids=[c[0] for c in engine_gpu.INTEGRATION])
def test_integration_tables(sweep_mode, cid, case):
    engine_gpu.test_integration_tables_gpu(cid, case)


@pytest.mark.parametrize("kw", [
    dict(n_nodes=10), dict(n_nodes=50), dict(n_nodes=100),
    dict(n_nodes=40, victim_queues=3, reclaimer_jobs=6, reclaimer_tasks=2, reclaimer_gpus=4.0),
    dict(n_nodes=64, running_per_node=6, victim_queues=2, reclaimer_jobs=20, reclaimer_tasks=1, reclaimer_gpus=2.0),
])
@pytest.mark.parametrize("action", ["reclaim", "consolidation"])
def test_solver_synthetic(sweep_mode, kw, action):
    engine_gpu.test_solver_synthetic(kw, action)


@pytest.mark.parametrize("chunk", range(8))
def test_cycle_fuzz(sweep_mode, chunk):
    cycle_fuzz.test_cycle_fuzz_engine_equals_oracle(chunk)


@pytest.mark.parametrize("name", [n for n in vr.REGIMES if n[0] in "ac"])
def test_value_regimes(sweep_mode, name):
    regime_gpu.test_regime_cycle_matches_oracle(name)


def _cycle_small_reclaim_sweeps():
    snap = synthetic.config_snapshot("config3-cycle-small")
    e = Engine()
    e.load(snap)
    e.run("allocate")
    r = e.run("reclaim")
    sweeps = e.stats().decisions
    evicted = int(r.pods_evicted)
    e.close()
    return sweeps, evicted


def test_cycle_small_reclaim_sweeps_on_the_host(monkeypatch):
    """config3-cycle-small: allocate leaves the cluster full, so every simulation's feasible set is a handful of
    victims' nodes; reclaim answers all of them on the host and launches no GPU simulation sweep."""
    monkeypatch.delenv("KAI_HOST_SWEEP_MAX", raising=False)
    monkeypatch.delenv("KAI_HOST_SWEEP_CHECK", raising=False)
    sweeps, evicted = _cycle_small_reclaim_sweeps()
    assert evicted > 0
    assert sweeps == 0
    monkeypatch.setenv("KAI_HOST_SWEEP_MAX", "0")
    sweeps_gpu, evicted_gpu = _cycle_small_reclaim_sweeps()
    assert sweeps_gpu > 0 and evicted_gpu == evicted
