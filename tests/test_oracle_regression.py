"""Digest regression of the oracle on the synthetic workloads the GPU parity tests use (CPU).

The engine is compared with the oracle on these snapshots on the GPU box; here the oracle's own outcome is pinned by a
digest recorded when engine and oracle last agreed on the GPU (tests/golden/oracle_digests.json), so that a change to the
oracle that would silently move it away from the engine is caught without a GPU.  Regenerate with
`python tests/test_oracle_regression.py --record` only together with a green `pytest -m gpu` run.
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kai_scheduler_b200 import abi, synthetic  # noqa: E402
from oracle_lib import Oracle  # noqa: E402

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_digests.json")


def _workloads():
    out = {}
    for i, kw in enumerate([
        dict(n_nodes=100, n_jobs=500, tasks_per_job=1, n_queues=10),
        dict(n_nodes=64, n_jobs=700, tasks_per_job=1, n_queues=4),
        dict(n_nodes=300, n_jobs=400, tasks_per_job=4, n_queues=12),
        dict(n_nodes=257, n_jobs=600, tasks_per_job=3, n_queues=7, mixed=True),
        dict(n_nodes=1000, n_jobs=3000, tasks_per_job=2, n_queues=40, mixed=True),
    ]):
        out[f"allocate-{i}"] = (synthetic.benchmark_snapshot(**kw), {}, ["allocate"])
    for name in ("reclaim-large-10", "reclaim-large-100", "cycle5-small", "config4-small", "config3-cycle-small"):
        out[name] = (synthetic.config_snapshot(name), {}, list(synthetic.CONFIG_ACTIONS.get(name, ["allocate"])))
    snap = synthetic.reclaim_snapshot(64, victim_queues=3, reclaimer_jobs=6, reclaimer_tasks=2, reclaimer_gpus=4.0)
    out["victims-all-actions"] = (snap, {}, ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"])
    snap = synthetic.reclaim_snapshot(64, victim_queues=3, reclaimer_jobs=6, reclaimer_tasks=2, reclaimer_gpus=4.0)
    rng = np.random.default_rng(7)
    snap.now_s = 50_000.0
    snap.job_last_start_s = snap.now_s - rng.choice(np.array([5.0, 50.0, 500.0, -1.0]), size=snap.n_jobs)
    snap.queue_reclaim_min_runtime_s = rng.choice(np.array([-1.0, 0.0, 20.0, 100.0]), size=snap.n_queues)
    snap.queue_preempt_min_runtime_s = rng.choice(np.array([-1.0, 10.0, 100.0]), size=snap.n_queues)
    out["victims-min-runtime"] = (snap, dict(default_reclaim_min_runtime_s=30.0, default_preempt_min_runtime_s=30.0), ["reclaim"])
    # the full-cycle workload of tests/test_engine_gpu.py (consolidation reaches the RemoveTask no-op, node_info.go:495-513)
    snap = synthetic.reclaim_snapshot(n_nodes=48, running_per_node=7, victim_queues=2, reclaimer_jobs=12, reclaimer_tasks=2,
                                      reclaimer_gpus=3.0)
    out["full-cycle-48"] = (snap, {}, ["allocate", "consolidation", "reclaim", "preempt"])
    snap = synthetic.benchmark_snapshot(n_nodes=48, n_jobs=700, tasks_per_job=1, n_queues=8)
    snap.queue_usage = np.random.default_rng(11).choice(np.array([0.0, 0.05, 0.125, 0.25, 0.5]), size=(3, snap.n_queues))
    out["usage-k2"] = (snap, dict(k_value=2.0), ["allocate"])
    snap = synthetic.reclaim_snapshot(32, victim_queues=2, reclaimer_jobs=4, reclaimer_tasks=2, reclaimer_gpus=2.0)
    snap.job_signature = (np.arange(snap.n_jobs) % 5).astype(np.int32)
    out["signatures"] = (snap, dict(use_scheduling_signatures=True), ["reclaim", "consolidation"])
    return out


def digest(snap, cfg_kw, actions):
    o = Oracle(abi.make_config(**cfg_kw))
    o.load(snap)
    h = hashlib.sha256()
    for a in actions:
        r = o.run(a)
        for arr in (r.task_node, r.task_status, r.visits, r.node_idle, r.node_releasing, r.queue_allocated,
                    np.round(r.queue_fair_share, 6)):
            h.update(np.ascontiguousarray(arr).tobytes())
        h.update(f"{a}:{int(r.pods_placed)}:{int(r.pods_evicted)}".encode())
    return h.hexdigest()


WORKLOADS = _workloads()


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_oracle_outcome_is_unchanged(name):
    recorded = json.load(open(DIGESTS))
    snap, cfg_kw, actions = WORKLOADS[name]
    assert digest(snap, cfg_kw, actions) == recorded[name], f"the oracle's outcome on {name} moved"


if __name__ == "__main__":
    if "--record" in sys.argv:
        json.dump({k: digest(*v) for k, v in sorted(WORKLOADS.items())}, open(DIGESTS, "w"), indent=1)
        print("recorded", len(WORKLOADS), "digests")
