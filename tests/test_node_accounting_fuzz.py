"""Node accounting invariant of the oracle under a whole cycle, on seeded random clusters (CPU only).

After every action the per-node Idle / Releasing vectors of the result must equal what the reference's NodeInfo arithmetic
gives for the final task table (pkg/scheduler/api/node_info/node_info.go:337-420 addTaskResources / removeTaskResources):

  * Allocated / Binding / Bound / Running / Releasing entries take their request out of Idle,
  * Releasing entries add it to Releasing, Pipelined entries take it out of Releasing,
  * a victim that was evicted on node A and pipelined on node B in the same session keeps TWO entries, Releasing on A and
    Pipelined on B (Statement.Pipeline with a different node adds the task to B and leaves A's entry alone,
    framework/statement.go:193-240); the result carries one (node, status) per task, so the entry on A is tracked here.
    A later action of the cycle can evict the Pipelined entry on B and move the task on to C: then A and B both keep a
    Releasing entry (one clone per node in NodeInfo.PodInfos, node_info.go:400-402 — not bounded by two).

The proportion plugin's per-queue Allocated / AllocatedNotPreemptible (open-session sum over allocated statuses plus the
Allocate / Deallocate event handlers, plugins/proportion/proportion.go:347-372, :440-500) must likewise equal the sum over
the final table's active-allocated tasks, accumulated up the queue's parent chain.

Evicting a Pipelined task is legal (activeAllocatedStatuses includes Pipelined, pod_status.go:66) and can drive Idle below
zero exactly as in the reference — the invariant is on the arithmetic, not on the sign.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dsl  # noqa: E402
from kai_scheduler_b200 import synthetic  # noqa: E402
from oracle_lib import Oracle  # noqa: E402
from test_snapshot_io import _random_topology  # noqa: E402

from kai_scheduler_b200 import abi  # noqa: E402

S = abi.POD_STATUS_NAMES
TAKES_IDLE = S["Allocated"] | S["Binding"] | S["Bound"] | S["Running"] | S["Releasing"]
ACTIVE_ALLOCATED = S["Allocated"] | S["Pipelined"] | S["Binding"] | S["Bound"] | S["Running"]
ACTIONS = ["allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"]


def _entries(status, node, ghosts):
    """(task, node, status) entries held by the nodes: one per placed task plus the Releasing leftovers of moved victims."""
    out = [(t, int(node[t]), int(status[t])) for t in range(len(status)) if node[t] >= 0 and (int(status[t]) & (TAKES_IDLE | S["Pipelined"]))]
    return out + [(t, n, S["Releasing"]) for t, n in ghosts]


def _account(base_free, base_rel, req, entries):
    idle, rel = base_free.copy(), base_rel.copy()
    for t, n, st in entries:
        if st & TAKES_IDLE:
            idle[:, n] -= req[t]
        if st == S["Releasing"]:
            rel[:, n] += req[t]
        elif st == S["Pipelined"]:
            rel[:, n] -= req[t]
    return idle, rel


@pytest.mark.parametrize("chunk", range(8))
def test_node_vectors_follow_the_task_table(chunk):
    for seed in range(chunk * 50, (chunk + 1) * 50):
        rng = np.random.default_rng(5000 + seed)
        snap, meta = dsl.build_snapshot(_random_topology(rng))
        req = np.asarray(snap.task_req, dtype=np.float64)
        status, node, ghosts = snap.task_status.copy(), snap.task_node.copy(), []
        # what the nodes offer before any session task is counted (allocatable minus foreign pods)
        zero = np.zeros_like(snap.node_idle)
        used, held = _account(zero, zero, req, _entries(status, node, ghosts))
        base_free, base_rel = snap.node_idle - used, snap.node_releasing - held
        task_job = np.zeros(snap.n_tasks, dtype=int)
        for j in range(snap.n_jobs):
            for ps in range(snap.job_podset_begin[j], snap.job_podset_begin[j + 1]):
                task_job[snap.podset_task_begin[ps]:snap.podset_task_begin[ps + 1]] = j
        o = Oracle(abi.make_config(allow_consolidating_reclaim=True, max_consolidation_preemptees=-1))
        o.load(snap)
        for act in ACTIONS:
            res = o.run(act)
            for t in range(len(status)):
                moved = node[t] >= 0 and res.task_node[t] != node[t] and (int(status[t]) & ACTIVE_ALLOCATED)
                if moved and int(res.task_status[t]) in (S["Pipelined"], S["Releasing"]):
                    ghosts.append((t, int(node[t])))
            status, node = res.task_status.copy(), res.task_node.copy()
            idle, rel = _account(base_free, base_rel, req, _entries(status, node, ghosts))
            np.testing.assert_allclose(res.node_idle, idle, rtol=0, atol=1e-9, err_msg=f"seed {seed} {act} idle")
            np.testing.assert_allclose(res.node_releasing, rel, rtol=0, atol=1e-9, err_msg=f"seed {seed} {act} releasing")
            alloc, fixed = np.zeros((3, snap.n_queues)), np.zeros((3, snap.n_queues))
            for t in np.flatnonzero(status & ACTIVE_ALLOCATED):
                j, q = task_job[t], int(snap.job_queue[task_job[t]])
                while q >= 0:
                    alloc[:, q] += req[t, :3]
                    if not int(snap.job_flags[j]) & abi.JOB_PREEMPTIBLE:
                        fixed[:, q] += req[t, :3]
                    q = int(snap.queue_parent[q])
            np.testing.assert_allclose(res.queue_allocated, alloc, rtol=0, atol=1e-9, err_msg=f"seed {seed} {act} queue allocated")
            np.testing.assert_allclose(res.queue_allocated_non_preemptible, fixed, rtol=0, atol=1e-9,
                                       err_msg=f"seed {seed} {act} queue non-preemptible")
        o.close()


VICTIM_WORKLOADS = [
    dict(n_nodes=8, running_per_node=6, victim_queues=3, reclaimer_jobs=4, reclaimer_tasks=2, reclaimer_gpus=3.0),
    dict(n_nodes=48, running_per_node=7, victim_queues=2, reclaimer_jobs=12, reclaimer_tasks=2, reclaimer_gpus=3.0),
    dict(n_nodes=64, running_per_node=7, victim_queues=3, reclaimer_jobs=20, reclaimer_tasks=3, reclaimer_gpus=2.0),
    dict(n_nodes=96, running_per_node=6, victim_queues=4, reclaimer_jobs=24, reclaimer_tasks=2, reclaimer_gpus=3.0),
    dict(n_nodes=24, running_per_node=6, victim_queues=3, reclaimer_jobs=20, reclaimer_tasks=3, reclaimer_gpus=3.0),
]


@pytest.mark.parametrize("kw", VICTIM_WORKLOADS, ids=[f"n{k['n_nodes']}q{k['victim_queues']}j{k['reclaimer_jobs']}" for k in VICTIM_WORKLOADS])
def test_moved_victims_keep_one_entry_per_node(kw):
    """Victim workloads where consolidation moves a victim (A -> B) and a later statement evicts it on B and re-places it
    on C: the task holds entries on three nodes (found on the GPU: oracle and engine both kept only two and disagreed).  The
    result carries one (node, status) per task, so the clones the nodes hold are read from the oracle (test-only export)
    and checked both ways: the node vectors follow from the entries, and every placed task of the result has its entry."""
    snap = synthetic.reclaim_snapshot(**kw)
    req = np.asarray(snap.task_req, dtype=np.float64)
    zero = np.zeros_like(snap.node_idle)
    used, held = _account(zero, zero, req, _entries(snap.task_status, snap.task_node, []))
    base_free, base_rel = snap.node_idle - used, snap.node_releasing - held
    o = Oracle()
    o.load(snap)
    most = 0
    for act in ("allocate", "consolidation", "reclaim", "preempt"):
        res = o.run(act)
        entries = o.node_entries()
        assert len(set((t, n) for t, n, _ in entries)) == len(entries), "one clone per (task, node)"
        idle, rel = _account(base_free, base_rel, req, entries)
        np.testing.assert_allclose(res.node_idle, idle, rtol=0, atol=1e-9, err_msg=f"{act} idle")
        np.testing.assert_allclose(res.node_releasing, rel, rtol=0, atol=1e-9, err_msg=f"{act} releasing")
        held_by = {(t, n): st for t, n, st in entries}
        for t in range(snap.n_tasks):
            st, n = int(res.task_status[t]), int(res.task_node[t])
            if n >= 0 and st & (TAKES_IDLE | S["Pipelined"]):
                assert held_by.get((t, n)) == st, f"{act}: task {t} is {st} on node {n}, the node holds {held_by.get((t, n))}"
        per_task = {}
        for t, n, st in entries:
            per_task[t] = per_task.get(t, 0) + 1
            if (t, n) != (t, int(res.task_node[t])):
                assert st == S["Releasing"], f"{act}: a left-behind clone of task {t} on node {n} has status {st}"
        most = max(most, max(per_task.values()))
    o.close()
    assert most >= 3, "the workload no longer reaches three clones of one task"
