"""Multi-GPU parity check (run under torchrun on a box with >= 2 GPUs; not collected by pytest):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
        tests/mgpu_check.py

Every rank shards the node rows, runs allocate through the C ABI and compares bindings / statuses / visiting order /
queue tables with the CPU oracle, and its own node rows with the oracle's node tables.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from kai_scheduler_b200 import abi, engine, synthetic  # noqa: E402
from oracle_lib import Oracle  # noqa: E402
import resident_lib  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.cuda.set_device(local)
    eng = engine.Engine(abi.make_config(device=local, shard_rank=rank, shard_count=world))
    handles = [eng.export_peer_handle() if rank == 0 else b""]
    dist.broadcast_object_list(handles, src=0)
    eng.wire_peers(handles * world)
    ok = True
    for kw in (dict(n_nodes=300, n_jobs=400, tasks_per_job=4, n_queues=12),
               dict(n_nodes=257, n_jobs=600, tasks_per_job=3, n_queues=7, mixed=True),
               dict(n_nodes=64, n_jobs=700, tasks_per_job=1, n_queues=4),
               dict(n_nodes=2000, n_jobs=6000, tasks_per_job=2, n_queues=40, mixed=True)):
        snap = synthetic.benchmark_snapshot(**kw)
        eng.load(snap)
        res = eng.run("allocate")
        o = Oracle()
        o.load(snap)
        ref = o.run("allocate")
        own = engine.shard_node_mask(snap.node_name_rank, world, rank)
        first, count = engine.shard_range(snap.n_nodes, world, rank)
        same = (np.array_equal(res.task_node, ref.task_node) and np.array_equal(res.task_status, ref.task_status)
                and np.array_equal(res.visits, ref.visits) and np.array_equal(res.queue_allocated, ref.queue_allocated)
                and first == rank and int(own.sum()) == count
                and np.array_equal(res.node_idle[:, own], ref.node_idle[:, own])
                and np.array_equal(res.node_releasing[:, own], ref.node_releasing[:, own]))
        print(f"rank {rank}/{world} {kw}: {'OK' if same else 'MISMATCH'} placed {res.pods_placed} sweeps {eng.stats().decisions}",
              flush=True)
        ok = ok and same
    # one whole cycle (allocate, consolidation, reclaim, preempt, stalegangeviction) on node-striped GPUs; the last
    # cluster has over-committed GPU nodes (negative idle GPUs): every rank's merged top-k list is cut at a negative key
    import value_regime as vr
    cycles = [(kw, synthetic.reclaim_snapshot(**kw)) for kw in (
        dict(n_nodes=48, running_per_node=7, victim_queues=2, reclaimer_jobs=12, reclaimer_tasks=2, reclaimer_gpus=3.0),
        dict(n_nodes=100), dict(n_nodes=333, running_per_node=8, victim_queues=3, reclaimer_jobs=9, reclaimer_tasks=3, reclaimer_gpus=4.0))]
    cycles.append(("overcommitted_gpus(333)", vr.overcommitted_gpus(333, 6, (1, 2, 3, 4, 8), stripes=(1, 3))))
    for kw, snap in cycles:
        eng.load(snap)
        o = Oracle()
        o.load(snap)
        own = engine.shard_node_mask(snap.node_name_rank, world, rank)
        for action in ("allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"):
            res, ref = eng.run(action), o.run(action)
            same = (np.array_equal(res.task_node, ref.task_node) and np.array_equal(res.task_status, ref.task_status)
                    and np.array_equal(res.visits, ref.visits) and np.array_equal(res.queue_allocated, ref.queue_allocated)
                    and res.pods_evicted == ref.pods_evicted
                    and np.array_equal(res.node_idle[:, own], ref.node_idle[:, own])
                    and np.array_equal(res.node_releasing[:, own], ref.node_releasing[:, own]))
            print(f"rank {rank}/{world} cycle {kw} {action}: {'OK' if same else 'MISMATCH'} placed {res.pods_placed} evicted {res.pods_evicted}", flush=True)
            ok = ok and same
    # non-round values (tests/value_regime.py): inexact node totals and queue sums must give every rank the oracle's bits
    for name in ("a_totals", "b_queues"):
        snap, _ = vr.regime(name)  # both regimes run with the default configuration
        eng.load(snap)
        res = eng.run("allocate")
        o = Oracle()
        o.load(snap)
        ref = o.run("allocate")
        own = engine.shard_node_mask(snap.node_name_rank, world, rank)
        same = (np.array_equal(res.task_node, ref.task_node) and np.array_equal(res.task_status, ref.task_status)
                and np.array_equal(res.visits, ref.visits) and np.array_equal(res.total_resource, ref.total_resource)
                and np.array_equal(res.queue_request, ref.queue_request)
                and np.array_equal(res.queue_allocated, ref.queue_allocated)
                and np.array_equal(res.queue_allocated_non_preemptible, ref.queue_allocated_non_preemptible)
                and np.array_equal(res.queue_fair_share, ref.queue_fair_share)
                and np.array_equal(res.node_idle[:, own], ref.node_idle[:, own]))
        print(f"rank {rank}/{world} value regime {name}: {'OK' if same else 'MISMATCH'} placed {res.pods_placed}", flush=True)
        ok = ok and same
        o.close()
    # topology-constrained gangs (config-4 shape) on node-striped GPUs
    for kw in (dict(n_nodes=512, n_gangs=60, nodes_per_rack=8, racks_per_leaf=4, leaves_per_spine=4, running_fraction=0.3),
               dict(n_nodes=2048, n_gangs=300)):
        snap = synthetic.topology_snapshot(**kw)
        eng.load(snap)
        res = eng.run("allocate")
        o = Oracle()
        o.load(snap)
        ref = o.run("allocate")
        own = engine.shard_node_mask(snap.node_name_rank, world, rank)
        same = (np.array_equal(res.task_node, ref.task_node) and np.array_equal(res.task_status, ref.task_status)
                and np.array_equal(res.visits, ref.visits) and np.array_equal(res.node_idle[:, own], ref.node_idle[:, own]))
        print(f"rank {rank}/{world} topology {kw}: {'OK' if same else 'MISMATCH'} placed {res.pods_placed}", flush=True)
        ok = ok and same
    # resident snapshot on node-striped GPUs (bench.py --gpus N reloads this way): cycles of tests/resident_lib.next_cycle,
    # the same structure_epoch every cycle.  Every rank simulates the same cycles (same seed, the oracle's outcome).
    for kw in (dict(n_nodes=48, running_per_node=7, victim_queues=2, reclaimer_jobs=12, reclaimer_tasks=2, reclaimer_gpus=3.0),
               dict(n_nodes=333, running_per_node=8, victim_queues=3, reclaimer_jobs=9, reclaimer_tasks=3, reclaimer_gpus=4.0)):
        rng = np.random.default_rng(kw["n_nodes"])
        snap = resident_lib.prepare(synthetic.reclaim_snapshot(**kw), rng)
        runner = resident_lib.ResidentRunner(lambda: eng)
        own = engine.shard_node_mask(snap.node_name_rank, world, rank)
        for cycle in range(4):
            runner.load(snap)
            o = Oracle()
            o.load(snap)
            same = True
            for action in ("allocate", "consolidation", "reclaim", "preempt", "stalegangeviction"):
                res, ref = eng.run(action), o.run(action)
                same = same and (np.array_equal(res.task_node, ref.task_node) and np.array_equal(res.task_status, ref.task_status)
                                 and np.array_equal(res.visits, ref.visits) and np.array_equal(res.queue_allocated, ref.queue_allocated)
                                 and np.allclose(res.queue_fair_share, ref.queue_fair_share, rtol=0, atol=1e-6) and res.pods_evicted == ref.pods_evicted
                                 and np.array_equal(res.node_idle[:, own], ref.node_idle[:, own])
                                 and np.array_equal(res.node_releasing[:, own], ref.node_releasing[:, own]))
            ok = ok and same
            print(f"rank {rank}/{world} resident n_nodes={kw['n_nodes']} cycle {cycle} (resident loads {runner.resident_loads}): "
                  f"{'OK' if same else 'MISMATCH'}", flush=True)
            o.close()
            snap = resident_lib.next_cycle(snap, ref, rng)
        ok = ok and runner.resident_loads == 3
    t = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("MGPU PARITY", "PASS" if int(t.item()) == 1 else "FAIL", flush=True)
    eng.close()
    dist.destroy_process_group()
    sys.exit(0 if int(t.item()) == 1 else 1)


if __name__ == "__main__":
    main()
