"""framework.Statement (statement.go:36-663) restated in the oracle, checked on the scenarios of statement_test.go
(CPU): Evict / Pipeline / Allocate, their undo, and the undo of an undo, on the reference's own fixture shapes
(`TestStatement_*`, whole-GPU cases; the fractional ones need GPU sharing).  The Go tests compare the task, the job's
Allocated and the node's Idle / Used / Releasing before and after; here the same quantities are the task status /
node, the queue's allocated GPUs and the node tables.
"""
import ctypes as C

import numpy as np
import pytest

import dsl
from kai_scheduler_b200 import abi
from oracle_lib import Oracle, lib

EVICT, PIPELINE, ALLOCATE, UNDO, DISCARD, PIPELINE_NO_UPDATE, ROLLBACK = 0, 1, 2, 3, 4, 5, 6


def session(jobs, gpus=2):
    topo = {"Nodes": {"node0": {"GPUs": gpus}}, "Queues": [{"Name": "queue0", "DeservedGPUs": gpus}], "Jobs": jobs}
    snap, meta = dsl.build_snapshot(topo)
    o = Oracle()
    o.load(snap)
    return o, snap, meta


def job(name, state, node=None, gpus=1):
    task = {"State": state}
    if node:
        task["NodeName"] = node
    return {"Name": name, "RequiredGPUsPerTask": gpus, "QueueName": "queue0", "Priority": 50, "Tasks": [task]}


def exercise(o, ops):
    ip = C.POINTER(C.c_int32)
    fn = lib().kai_oracle_statement_exercise
    fn.argtypes = [C.c_void_p, C.c_int, ip, ip, ip]
    k = np.array([x[0] for x in ops], dtype=np.int32)
    t = np.array([x[1] for x in ops], dtype=np.int32)
    n = np.array([x[2] if len(x) > 2 else -1 for x in ops], dtype=np.int32)
    return fn(o._h, len(ops), k.ctypes.data_as(ip), t.ctypes.data_as(ip), n.ctypes.data_as(ip))


def state(o):
    r = o.fair_share()
    return (r.task_status.tolist(), r.task_node.tolist(), r.node_idle[2].tolist(), r.node_releasing[2].tolist(),
            r.queue_allocated[2].tolist(), r.node_idle[3].tolist())


def test_evict_then_unevict_restores_everything():  # TestStatement_Evict_Unevict (:27-154)
    o, _, _ = session([job("running_job0", "Running", "node0")])
    before = state(o)
    assert exercise(o, [(EVICT, 0), (UNDO, 0)]) == 2
    assert state(o) == before
    assert before[4][0] == 1 and before[2] == [1.0]  # jobGpuAllocation 1, one of two GPUs used


def test_evict():  # TestStatement_Evict (:156-305)
    o, _, _ = session([job("pending_job0", "Pending")])
    assert exercise(o, [(EVICT, 0)]) < 0  # "node doesn't exist in session": a Pending pod cannot be evicted
    o, _, _ = session([job("running_job0", "Running", "node0")])
    before = state(o)
    assert exercise(o, [(EVICT, 0)]) == 1
    st, node, idle, rel, qalloc, idle_pods = state(o)
    assert st == [abi.POD_RELEASING] and node == [0]
    assert idle == before[2] and rel == [1.0]      # still Used on the node, now also Releasing
    assert qalloc[0] == 0.0                        # proportion's deallocate handler ran (statement.go:101-110)


def test_evict_undo_undo():  # TestStatement_Evict_Undo_Undo (:307-460): undoing the undo evicts again
    o, _, _ = session([job("running_job0", "Running", "node0")])
    exercise(o, [(EVICT, 0)])
    evicted = state(o)
    assert exercise(o, [(UNDO, 0), (UNDO, 1)]) == 4  # evict, undo, evict again (the redo), undo
    assert state(o) == evicted


def test_pipeline_then_unpipeline_restores_everything():  # TestStatement_Pipeline_Unpipeline (:462-693)
    o, _, _ = session([job("releasing_job0", "Releasing", "node0"), job("pending_job0", "Pending")], gpus=1)
    before = state(o)
    assert exercise(o, [(PIPELINE, 1, 0), (UNDO, 0)]) == 2
    assert state(o) == before


def test_pipeline():  # TestStatement_Pipeline (:695-822): the pod takes the releasing GPU
    o, _, _ = session([job("releasing_job0", "Releasing", "node0"), job("pending_job0", "Pending")], gpus=1)
    before = state(o)
    assert before[3] == [1.0] and before[2] == [0.0]
    assert exercise(o, [(PIPELINE, 1, 0)]) == 1
    st, node, idle, rel, qalloc, _ = state(o)
    assert st == [abi.POD_RELEASING, abi.POD_PIPELINED] and node == [0, 0]
    assert idle == [0.0] and rel == [0.0]          # Releasing -= request (node_info.go:483-488)
    assert qalloc[0] == before[4][0] + 1


def test_pipeline_undo_undo():  # TestStatement_Pipeline_Undo_Undo (:824-958)
    o, _, _ = session([job("releasing_job0", "Releasing", "node0"), job("pending_job0", "Pending")], gpus=1)
    exercise(o, [(PIPELINE, 1, 0)])
    pipelined = state(o)
    assert exercise(o, [(UNDO, 0), (UNDO, 1)]) == 4  # evict, undo, evict again (the redo), undo
    assert state(o) == pipelined


def test_allocate_then_unallocate_restores_everything():  # TestStatement_Allocate_Unallocate (:960-1064)
    o, _, _ = session([job("pending_job0", "Pending")])
    before = state(o)
    assert exercise(o, [(ALLOCATE, 0, 0), (UNDO, 0)]) == 2
    assert state(o) == before


def test_allocate():  # TestStatement_Allocate (:1066-1170)
    o, _, _ = session([job("pending_job0", "Pending")])
    assert exercise(o, [(ALLOCATE, 0, 0)]) == 1
    st, node, idle, rel, qalloc, idle_pods = state(o)
    assert st == [abi.POD_ALLOCATED] and node == [0] and idle == [1.0] and rel == [0.0] and qalloc[0] == 1.0
    assert idle_pods == [109.0]


def test_allocate_undo_undo():  # TestStatement_Allocate_Undo_Undo (:1172-1282)
    o, _, _ = session([job("pending_job0", "Pending")])
    exercise(o, [(ALLOCATE, 0, 0)])
    allocated = state(o)
    assert exercise(o, [(UNDO, 0), (UNDO, 1)]) == 4  # evict, undo, evict again (the redo), undo
    assert state(o) == allocated


# statement_checkpoint_test.go:30-230 TestStatement_Checkpoint: running_job0 (task 1 after the DSL's priority sort keeps
# the order: both priority 50 -> running_job0-0 = task 0, pending_job0-0 = task 1) on node0 with 2 GPUs; every sequence
# is followed by Rollback(checkpoint 0) and must leave jobs and nodes as they were
RUN_T, PEND_T = 0, 1
CHECKPOINT = [
    ("rollback evict", [(EVICT, RUN_T)]),
    ("rollback allocate", [(ALLOCATE, PEND_T, 0)]),
    ("rollback pipeline updateIfNeeded true", [(PIPELINE, PEND_T, 0)]),
    ("rollback pipeline updateIfNeeded false", [(PIPELINE_NO_UPDATE, PEND_T, 0)]),
    ("rollback allocate evict", [(ALLOCATE, PEND_T, 0), (EVICT, PEND_T)]),
    ("rollback pipeline evict", [(PIPELINE, PEND_T, 0), (EVICT, PEND_T)]),
    ("rollback evict pipeline", [(EVICT, RUN_T), (PIPELINE, RUN_T, 0)]),
    ("rollback pipeline evict update false", [(PIPELINE_NO_UPDATE, PEND_T, 0), (EVICT, PEND_T)]),
    ("rollback evict pipeline update false", [(EVICT, RUN_T), (PIPELINE_NO_UPDATE, RUN_T, 0)]),
    ("rollback evict checkpoint pipeline update false", [(EVICT, RUN_T), (PIPELINE_NO_UPDATE, RUN_T, 0), (ROLLBACK, 1)]),
]


@pytest.mark.parametrize("name,ops", CHECKPOINT, ids=[c[0] for c in CHECKPOINT])
def test_statement_checkpoint_rollback(name, ops):
    o, _, meta = session([job("running_job0", "Running", "node0"), job("pending_job0", "Pending")])
    assert meta["task_names"] == ["running_job0-0", "pending_job0-0"]
    before = state(o)
    assert exercise(o, ops) >= 1
    assert exercise(o, [(ROLLBACK, 0)]) >= 0
    assert state(o) == before


def test_one_clone_per_node_is_unbounded():
    """NodeInfo.PodInfos is a map per node (node_info.go:400-402): a pod that is evicted on A, pipelined to B, evicted
    there and pipelined to C holds a clone on each of the three nodes (Releasing, Releasing, Pipelined); Discard walks
    back through all of them.  (Round 2: oracle and engine used to keep two entries and disagreed.)"""
    topo = {"Nodes": {f"node{i}": {"GPUs": 2} for i in range(3)}, "Queues": [{"Name": "queue0", "DeservedGPUs": 6}],
            "Jobs": [job("running_job0", "Running", "node0")]}
    snap, _ = dsl.build_snapshot(topo)
    o = Oracle()
    o.load(snap)
    before = state(o)
    S = abi.POD_STATUS_NAMES
    assert o.node_entries() == [(0, 0, S["Running"])]
    assert exercise(o, [(EVICT, 0), (PIPELINE, 0, 1), (EVICT, 0), (PIPELINE, 0, 2)]) == 4
    assert sorted(o.node_entries()) == [(0, 0, S["Releasing"]), (0, 1, S["Releasing"]), (0, 2, S["Pipelined"])]
    r = o.fair_share()
    # node0: the original pod is Releasing (its GPU still taken, counted as releasing); node1: an evicted Pipelined clone
    # takes a GPU out of Idle and adds it to Releasing (pod_status.go:66: Pipelined is active-allocated, so it can be
    # evicted); node2: the Pipelined clone takes the GPU out of Releasing
    assert r.node_idle[2].tolist() == [1.0, 1.0, 2.0] and r.node_releasing[2].tolist() == [1.0, 1.0, -1.0]
    assert exercise(o, [(DISCARD, 0)]) == 0
    assert state(o) == before and o.node_entries() == [(0, 0, S["Running"])]
