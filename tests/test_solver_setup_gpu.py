"""Solver set-up from the prepare kernels, engine-kept scratch and the flat victims queues (GPU box).

The solver takes its per-podset active-allocated and pending counts from k_prep_jobs instead of scanning every task
status, keeps its per-node / per-job / per-task scratch on the engine between actions (invalidated by epoch stamps),
reconciles task slots only over the tasks an action changed, and keeps every JobsOrder heap in one arena.  Every
solver workload of the GPU suite runs here with KAI_SOLVER_SETUP_CHECK=1, which recounts the podset and pending-job
counts by scanning every task status and fails the action on any difference, two ways, each bit for bit against the
oracle:
  * "cache":    the default victims-queue cache (per-leaf runs, lazily loaded leaves, copies of the first build);
  * "no-cache": KAI_NO_VICTIM_CACHE=1, every victims queue built from all jobs (the reference's own construction).
The workloads cover releasing-only and not-ready nodes, multi-podset and elastic jobs below, at and above
minAvailable, non-preemptible jobs, leaf queues without an eligible victim, consolidation then reclaim in one session
(integration tables) and resident reload cycles where N, J and T stay the same next to full loads where they change.
"""
import pytest

import test_cycle_fuzz_gpu as cycle_fuzz
import test_engine_gpu as engine_gpu
import test_resident_gpu as resident_gpu
import test_value_regime_gpu as regime_gpu
import value_regime as vr

pytestmark = pytest.mark.gpu

MODES = {
    "cache": {"KAI_SOLVER_SETUP_CHECK": "1"},
    "no-cache": {"KAI_SOLVER_SETUP_CHECK": "1", "KAI_NO_VICTIM_CACHE": "1"},
}


@pytest.fixture(params=sorted(MODES))
def setup_mode(request, monkeypatch):
    monkeypatch.delenv("KAI_NO_VICTIM_CACHE", raising=False)
    for k, v in MODES[request.param].items():
        monkeypatch.setenv(k, v)
    return request.param


@pytest.mark.parametrize("cid,case", engine_gpu.SOLVER, ids=[c[0] for c in engine_gpu.SOLVER])
def test_solver_tables(setup_mode, cid, case):
    engine_gpu.test_solver_tables_gpu(cid, case)


@pytest.mark.parametrize("cid,case", engine_gpu.INTEGRATION, ids=[c[0] for c in engine_gpu.INTEGRATION])
def test_integration_tables(setup_mode, cid, case):
    engine_gpu.test_integration_tables_gpu(cid, case)


@pytest.mark.parametrize("kw", [
    dict(n_nodes=10), dict(n_nodes=50), dict(n_nodes=100),
    dict(n_nodes=40, victim_queues=3, reclaimer_jobs=6, reclaimer_tasks=2, reclaimer_gpus=4.0),
    dict(n_nodes=64, running_per_node=6, victim_queues=2, reclaimer_jobs=20, reclaimer_tasks=1, reclaimer_gpus=2.0),
])
@pytest.mark.parametrize("action", ["reclaim", "consolidation"])
def test_solver_synthetic(setup_mode, kw, action):
    engine_gpu.test_solver_synthetic(kw, action)


@pytest.mark.parametrize("chunk", range(8))
def test_cycle_fuzz(setup_mode, chunk):
    cycle_fuzz.test_cycle_fuzz_engine_equals_oracle(chunk)


@pytest.mark.parametrize("name", [n for n in vr.REGIMES if n[0] == "a"])
def test_value_regime_a(setup_mode, name):
    regime_gpu.test_regime_cycle_matches_oracle(name)


def test_resident_integration_tables(setup_mode):
    """One engine per table over resident reloads (same N, J, T) and full loads: the engine-kept scratch."""
    resident_gpu.test_integration_tables_on_one_resident_engine()


@pytest.mark.parametrize("chunk", range(2))
def test_resident_random_clusters(setup_mode, chunk):
    resident_gpu.test_resident_cycles_random_clusters(chunk)


def test_shape_change_reloads(setup_mode):
    """A full load that changes the snapshot's shape resizes the scratch."""
    resident_gpu.test_shape_change_under_the_same_epoch_loads_in_full()
