"""Non-round resource values for the engine-vs-oracle parity tests (test_value_regime.py, test_value_regime_gpu.py).

The synthetic and DSL clusters use round quantities (2e7 mCPU / 2e10 B nodes, 1000 mCPU / 1e9 B pods, integer GPUs).
On such data every f64 sum on the scheduling path is exact, so it has the same bits in any order and association, and
a kernel that sums in another order than the oracle (DESIGN.md §2) or reassociates a formula still matches.  The
generators here keep the structure of those shapes and rewrite their values into realistic, non-round Kubernetes
quantities (arbitrary milli-CPU, memory in Ki multiples, odd byte counts), in four regimes, plus (e) with negative
Idle GPUs:

  (a) inexact_totals      >= 5 000 ~2 TB nodes, each with a foreign pod of an odd byte count: the memory total passes
                          2^53 at a granularity of 1 B, so the order of the node sum decides its bits.
  (b) inexact_queue_sums  >= 10 000 running / pending tasks of ~3e12 + odd B under one department: queue_request,
                          queue_allocated and queue_allocated_non_preemptible of the ancestors are inexact sums.
  (c) score_near_ties     CPU-only pods on CPU-only nodes whose Idle CPU differs by a few milli next to one far
                          larger node: binpack / spread scores differ in the last bits or tie (the name rank decides);
                          plus the edges mn == mx, mx == 0 and overall == 0.
  (d) fractional_shares   non-integer k_value, historical usage, over-quota weights, deserved quotas and CPU totals.
  (e) overcommitted_gpus  nodes whose running pods hold more GPUs than the node has: negative Idle GPUs, which the
                          idle-GPU filter's top-k list must order below zero (and -0.0 rows equal to +0.0 ones).

It also holds the exact references the CPU tests use: Fraction sums, the sequential rounding bound, a numpy emulation
of k_node_totals' reduction order, and a restatement of SetResourcesShare that reports which paths it took.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from kai_scheduler_b200 import abi, synthetic

U = 2.0 ** -53          # unit roundoff of binary64
H100_SMS = 132          # SM count of an H100 SXM: k_node_totals' grid is min(4 * SMs, ceil(N / 256)) blocks of 256
ACTIONS = ("allocate", "consolidation", "reclaim", "preempt", "stalegangeviction")


def _ki(rng, lo_bytes: float, hi_bytes: float, size) -> np.ndarray:
    return rng.integers(int(lo_bytes) // 1024, int(hi_bytes) // 1024, size=size).astype(np.float64) * 1024.0


def _odd(rng, lo: float, hi: float, size) -> np.ndarray:
    return (rng.integers(int(lo) // 2, int(hi) // 2, size=size) * 2 + 1).astype(np.float64)


def refresh_node_tables(snap: abi.Snapshot) -> abi.Snapshot:
    """Idle / Releasing from Allocatable, the foreign pods and the tasks placed on each node (dsl.build_snapshot's
    rules: Releasing tasks count as releasing, Pipelined ones give releasing back, the rest use idle)."""
    alloc = snap.node_allocatable
    idle = alloc.copy()
    rel = np.zeros_like(alloc)
    if snap.node_foreign is not None:
        idle[:3] -= snap.node_foreign
    for t in np.flatnonzero(snap.task_node >= 0):
        n, st, req = int(snap.task_node[t]), int(snap.task_status[t]), snap.task_req[t]
        if st == abi.POD_RELEASING:
            rel[:, n] += req
            idle[:, n] -= req
        elif st == abi.POD_PIPELINED:
            rel[:, n] -= req
        else:
            idle[:, n] -= req
    snap.node_idle, snap.node_releasing = idle, rel
    return snap


def _run_on_nodes(snap: abi.Snapshot, jobs, nodes) -> None:
    """Marks every task of `jobs` Running, job k's tasks on nodes[k]."""
    for j, n in zip(jobs, nodes):
        for ps in range(snap.job_podset_begin[j], snap.job_podset_begin[j + 1]):
            t0, t1 = snap.podset_task_begin[ps], snap.podset_task_begin[ps + 1]
            snap.task_status[t0:t1] = abi.POD_RUNNING
            snap.task_node[t0:t1] = n


# ------------------------------------------------------------------------------------------------------------------
# the regimes
# ------------------------------------------------------------------------------------------------------------------
def inexact_totals(n_nodes: int = 5000, seed: int = 1, mem_tb: tuple = (1.9, 2.2)) -> abi.Snapshot:
    """(a) benchmark shape with request mix; nodes of `mem_tb` TB in Ki multiples, arbitrary milli-CPU, one foreign pod
    of an odd byte count per node, a few NotReady nodes, one running pod on each of the first nodes."""
    rng = np.random.default_rng(seed)
    snap = synthetic.benchmark_snapshot(n_nodes=n_nodes, n_jobs=n_nodes // 2, tasks_per_job=2, n_queues=8, mixed=True,
                                        seed=seed)
    N, T = n_nodes, snap.n_tasks
    snap.node_allocatable[0] = rng.integers(96_000, 256_000, size=N)             # e.g. 191937m
    snap.node_allocatable[1] = _ki(rng, mem_tb[0] * 1e12, mem_tb[1] * 1e12, N)
    foreign = np.zeros((3, N))
    foreign[0] = rng.integers(1, 4000, size=N)
    foreign[1] = _odd(rng, 1e8, 4e9, N)
    snap.node_foreign = foreign
    snap.task_req[:, 0] = rng.integers(50, 8000, size=T)
    snap.task_req[:, 1] = _odd(rng, 2e8, 64e9, T)
    snap.node_flags[rng.choice(N, size=N // 100, replace=False)] &= ~np.uint32(abi.NODE_READY)
    running = np.arange(0, snap.n_jobs, 4)        # one job in four runs, each on its own node (both tasks)
    running = running[snap.task_req[snap.podset_task_begin[running], 2] <= 4]
    _run_on_nodes(snap, running, np.arange(len(running)))
    return refresh_node_tables(snap)


def inexact_queue_sums(n_tasks: int = 10_000, seed: int = 2) -> abi.Snapshot:
    """(b) 8-task gangs in 4 leaf queues of one department; tasks of ~3e12 + odd B (so that even the
    non-preemptible running tasks' sum passes 2^53), two jobs in three non-preemptible; half the gangs run (one per
    node, in queues 0 and 2, over their deserved GPUs), the other half are pending and only 60 % of them fit on the
    free nodes, so reclaim has work left."""
    rng = np.random.default_rng(seed)
    n_jobs = n_tasks // 8
    snap = synthetic.benchmark_snapshot(n_nodes=n_jobs * 4 // 5, n_jobs=n_jobs, tasks_per_job=8, n_queues=4,
                                        named_depts=False)
    N, T = snap.n_nodes, snap.n_tasks
    snap.node_allocatable[0] = rng.integers(200_000, 400_000, size=N)
    snap.node_allocatable[1] = _ki(rng, 25.8e12, 27.6e12, N)
    snap.task_req[:, 0] = rng.integers(100, 20_000, size=T)
    snap.task_req[:, 1] = 3e12 + _odd(rng, 1, 2e11, T)
    snap.job_flags[np.arange(n_jobs) % 3 != 0] &= ~np.uint32(abi.JOB_PREEMPTIBLE)
    running = np.arange(0, n_jobs, 2)
    _run_on_nodes(snap, running, np.arange(len(running)))
    return refresh_node_tables(snap)


def score_near_ties(n_nodes: int = 96, seed: int = 3, wide: float = 2.0 ** 47) -> abi.Snapshot:
    """(c) CPU-only: no node has a GPU, no pod asks for one.  Idle CPU = a base + 0..3 milli (so scores tie exactly or
    differ by a few ulps) on every node but eight: one whose Idle CPU is `wide` milli larger and seven in between; the
    pods are small enough that every placement keeps the spread of Idle values."""
    rng = np.random.default_rng(seed)
    snap = synthetic.benchmark_snapshot(n_nodes=n_nodes, n_jobs=3 * n_nodes, tasks_per_job=1, n_queues=4)
    N, T = n_nodes, snap.n_tasks
    snap.node_allocatable[2] = 0.0
    snap.node_gpu_count = np.zeros(N)
    base = (64_000 + rng.integers(0, 4, size=N)).astype(np.float64)
    base[N // 3] += wide
    base[N // 3 + 1:N // 3 + 8] += np.floor(wide * np.arange(1, 8) / 9)   # mid-range scores, where equal forms round apart
    snap.node_allocatable[0] = base
    snap.node_allocatable[1] = _ki(rng, 5e11, 5e11 + 4096, N)
    snap.task_req[:, 2] = 0.0
    snap.task_req[:, 0] = rng.choice(np.array([1.0, 2.0, 3.0]), size=T)
    snap.task_req[:, 1] = _odd(rng, 1e6, 1e8, T)
    snap.queue_deserved[2] = -1.0
    snap.queue_oqw[2] = 1.0
    return refresh_node_tables(snap)


def score_edges(seed: int = 4) -> abi.Snapshot:
    """(c) edges of pack.go:45-64: mn == mx (every node the same Idle CPU), mx == 0 and overall == 0 (nodes without
    allocatable CPU and pods that ask for none), next to GPU nodes without GPUs left."""
    rng = np.random.default_rng(seed)
    snap = synthetic.benchmark_snapshot(n_nodes=24, n_jobs=60, tasks_per_job=1, n_queues=4)
    N, T = snap.n_nodes, snap.n_tasks
    snap.node_allocatable[2, :16] = 0.0                # 16 CPU-only nodes ...
    snap.node_allocatable[0, :8] = 0.0                 # ... 8 of them without any CPU (overall == 0, mx == 0)
    snap.node_allocatable[0, 8:16] = 77_777.0          # ... 8 with the same CPU (mn == mx)
    snap.node_allocatable[1] = _ki(rng, 1e11, 2e11, N)
    snap.node_gpu_count = snap.node_allocatable[2].copy()
    snap.task_req[:, 2] = np.where(np.arange(T) % 3 == 0, 1.0, 0.0)
    snap.task_req[:, 0] = np.where(np.arange(T) % 2 == 0, 0.0, 1001.0)
    snap.task_req[:, 1] = _odd(rng, 1e6, 1e9, T)
    return refresh_node_tables(snap)


def fractional_shares(seed: int = 5):
    """(d) over-subscribed queues with fractional historical usage, non-integer over-quota weights and deserved GPUs,
    and CPU quantities in micro-cores (non-integer milli): returns (snapshot, k_value)."""
    rng = np.random.default_rng(seed)
    snap = synthetic.benchmark_snapshot(n_nodes=16, n_jobs=200, tasks_per_job=1, n_queues=8)
    Q, N = snap.n_queues, snap.n_nodes
    snap.queue_usage = rng.random((3, Q)) * 0.4
    snap.queue_oqw = np.round(rng.uniform(0.2, 3.0, size=(3, Q)), 3)
    snap.queue_deserved = snap.queue_deserved.copy()
    snap.queue_deserved[2, :8] = np.round(rng.uniform(3.0, 17.0, size=8), 2)
    snap.queue_deserved[0, :8] = np.round(rng.uniform(1e5, 9e5, size=8), 3)
    foreign = np.zeros((3, N))
    foreign[0] = rng.integers(1, 4000, size=N) + 0.25 * rng.integers(0, 4, size=N)   # e.g. 1250.5m = 1250500u
    foreign[0, 0] += 0.125                                                          # the CPU total is not an integer
    foreign[1] = _odd(rng, 1e6, 1e9, N)
    snap.node_foreign = foreign
    snap.task_req[:, 0] = rng.integers(50, 4000, size=snap.n_tasks)
    snap.task_req[:, 1] = _odd(rng, 1e8, 4e9, snap.n_tasks)
    return refresh_node_tables(snap), 0.37


def _trim_gangs(snap: abi.Snapshot, n_run: int, sizes) -> abi.Snapshot:
    """Cuts reclaim_snapshot's equal reclaimer gangs (jobs after the n_run 1-task victims) to `sizes` tasks each."""
    top = int(max(sizes))
    keep = np.ones(snap.n_tasks, dtype=bool)
    for g, size in enumerate(sizes):
        keep[n_run + g * top + size:n_run + (g + 1) * top] = False
    snap.task_status, snap.task_node = snap.task_status[keep], snap.task_node[keep]
    snap.task_req = snap.task_req[keep]
    snap.task_order_rank = np.concatenate(
        [snap.task_order_rank[:n_run]] + [synthetic._name_rank("", size) for size in sizes]).astype(np.int32)
    snap.podset_min_available = np.concatenate([np.ones(n_run), np.asarray(sizes)]).astype(np.int32)
    snap.podset_task_begin = np.concatenate([np.arange(n_run), n_run + np.cumsum([0] + list(sizes))]).astype(np.int32)
    return snap


def overcommitted_gpus(n_nodes: int, running_per_node: int, gang_sizes, stripes=(1,), preemptible_every: int = 1,
                       seed: int = 7) -> abi.Snapshot:
    """(e) Over-committed GPU nodes: nodes whose GPU allocatable fell below the GPUs their running pods hold (a
    device-plugin restart or a GPU marked unhealthy), so Idle GPUs = -1..-3 (node_info.go addTask subtracts without a fit
    check and nothing clamps it).  Base: reclaim_snapshot with `running_per_node` running 1-GPU pods per node in two
    victim queues (deserved 0) and pending gangs of `gang_sizes` 8-GPU tasks in the reclaimer queue; the running pods
    are preemptible on every `preemptible_every`-th node only (fewer candidate victims keep the oracle's search short).

    Over-committed: every node of the name-rank stripes rank % 4 in `stripes` but the first three of each (a scanner of
    a 4- or 256-scanner grid holds ranks j * nscan + my, so its 4th candidate is negative and it has more rows), plus
    one node in 24 elsewhere.  Edge rows: a Releasing pod on an over-committed node (Idle < 0, Releasing > 0), a
    Pipelined pod (Releasing < 0), two nodes with no GPU allocatable and pods still running, and ten full nodes in
    interleaved name ranks, five with Idle and Releasing GPUs +0.0 and five with -0.0.  Three nodes are empty: no gang
    fits on them alone, but they count in the filter's top-k, so a list that drops them prunes scenarios the oracle
    simulates."""
    rng = np.random.default_rng(seed)
    snap = synthetic.reclaim_snapshot(n_nodes, running_per_node=running_per_node, victim_queues=2,
                                      reclaimer_jobs=len(gang_sizes), reclaimer_tasks=int(max(gang_sizes)), reclaimer_gpus=8.0)
    N, n_run, G = n_nodes, n_nodes * running_per_node, abi.RES_GPU
    snap = _trim_gangs(snap, n_run, gang_sizes)
    snap.job_flags[:n_run][snap.task_node[:n_run] % preemptible_every != 0] &= ~np.uint32(abi.JOB_PREEMPTIBLE)
    rank_to_node = np.argsort(snap.node_name_rank)
    over = np.zeros(N, dtype=bool)
    for st in stripes:
        over[rank_to_node[st + 4 * 3::4]] = True
    free = np.flatnonzero(~over)
    over[rng.choice(free, size=max(1, N // 24), replace=False)] = True
    snap.node_allocatable[G, over] = running_per_node - rng.integers(1, 4, size=int(over.sum()))
    rest = rank_to_node[[r for r in range(N) if not over[rank_to_node[r]]]]   # not over-committed, in name-rank order
    zero_alloc, minus_zero, plus_zero = rest[[3, len(rest) // 2]], rest[[5, 9, 13, 17, 21]], rest[[7, 11, 15, 19, 23]]
    snap.node_allocatable[G, zero_alloc] = 0.0
    snap.node_allocatable[G, np.concatenate([minus_zero, plus_zero])] = running_per_node
    free = rest[[27, len(rest) // 3, 2 * len(rest) // 3 + 1]]   # every pod on them finished: Idle = 8
    done = np.flatnonzero(np.isin(snap.task_node[:n_run], free))
    snap.task_status[done] = abi.POD_STATUS_NAMES["Succeeded"]
    snap.task_node[done] = -1
    on_over = np.flatnonzero(over[snap.task_node[:n_run]])
    snap.task_status[on_over[0]] = abi.POD_RELEASING
    snap.task_status[on_over[-1]] = abi.POD_PIPELINED
    snap = refresh_node_tables(snap)
    snap.node_idle[G, minus_zero] = -0.0
    snap.node_releasing[G, minus_zero] = -0.0
    return snap


def regime(name: str):
    """(snapshot, config) of a named regime."""
    if name == "e_overcommit":  # one row per scanner of the default grid; the largest gang needs more rows than are >= 0
        return overcommitted_gpus(96, 6, (4, 5, 6, 50), stripes=(1, 3)), abi.make_config()
    if name == "e_overcommit_2048":  # > 256 rows with free GPUs: even the default mode lists them on the GPU
        return overcommitted_gpus(2048, 6, (4, 5, 6, 8), preemptible_every=8), abi.make_config()
    if name == "a_totals":
        return inexact_totals(), abi.make_config()
    if name == "a_totals_1800":  # fits one node tile of a 2-CTA grid; ~5.4 TB nodes still pass 2^53 in total
        return inexact_totals(n_nodes=1800, seed=6, mem_tb=(5.2, 5.6)), abi.make_config()
    if name == "b_queues":
        return inexact_queue_sums(), abi.make_config()
    if name == "c_binpack":
        return score_near_ties(), abi.make_config()
    if name == "c_spread":
        return score_near_ties(), abi.make_config(gpu_placement=abi.PLACEMENT_SPREAD, cpu_placement=abi.PLACEMENT_SPREAD)
    if name == "c_edges":
        return score_edges(), abi.make_config()
    if name == "c_edges_spread":
        return score_edges(), abi.make_config(gpu_placement=abi.PLACEMENT_SPREAD, cpu_placement=abi.PLACEMENT_SPREAD)
    if name == "d_shares":
        snap, k = fractional_shares()
        return snap, abi.make_config(k_value=k)
    raise KeyError(name)


REGIMES = ("a_totals", "a_totals_1800", "b_queues", "c_binpack", "c_spread", "c_edges", "c_edges_spread", "d_shares",
           "e_overcommit", "e_overcommit_2048")


def idle_gpu_key(snap: abi.Snapshot) -> np.ndarray:
    """Idle + Releasing GPUs per node: the key of the idle-GPU scenario filter's top-k list."""
    return snap.node_idle[abi.RES_GPU] + snap.node_releasing[abi.RES_GPU]


def stripe_cut_goes_negative(snap: abi.Snapshot, nscan: int) -> bool:
    """Some scanner of an `nscan`-scanner grid (one GPU: ranks j * nscan + my) holds >= 5 rows of which at most 3 have
    a key >= 0: its 4th listed candidate is negative while it has more rows, so the list is cut at a negative key."""
    key_by_rank = idle_gpu_key(snap)[np.argsort(snap.node_name_rank)]
    return any(len(key_by_rank[my::nscan]) >= 5 and (key_by_rank[my::nscan] >= 0).sum() <= 3 for my in range(nscan))


def without_pending(snap: abi.Snapshot) -> abi.Snapshot:
    """The same cluster with every pending task marked Succeeded: no action has anything to do, so the totals and
    queue tables an engine reports come straight from the open-session kernels."""
    import copy
    s = copy.copy(snap)
    s.task_status = np.where(snap.task_status == abi.POD_PENDING, abi.POD_STATUS_NAMES["Succeeded"],
                             snap.task_status).astype(np.int32)
    return s


# ------------------------------------------------------------------------------------------------------------------
# exact references
# ------------------------------------------------------------------------------------------------------------------
def binpack_sweeps(snap: abi.Snapshot, res: abi.Result):
    """Replays an allocate of one-task CPU-only jobs in the oracle's visiting order: every sweep scores the fitting nodes
    with the oracle's own pack.go:45-64 (kai_oracle_binpack_score) plus the +100 / +10 terms of the NodeOrderFn sum.
    Returns (winner - runner-up in ulps of the winner per sweep, sweeps whose winner is not the oracle's node)."""
    from oracle_lib import lib
    f = lib().kai_oracle_binpack_score
    idle, rel, A = snap.node_idle.copy(), snap.node_releasing, snap.node_allocatable[abi.RES_CPU]
    gaps, mismatches = [], 0
    for j, _ in res.visits:
        t = snap.podset_task_begin[snap.job_podset_begin[j]]
        if res.task_node[t] < 0:
            continue
        req = snap.task_req[t]
        fit = (idle >= req[:, None]).all(axis=0)
        cur = idle[abi.RES_CPU] + rel[abi.RES_CPU]
        mn, mx = cur[A != 0].min(), cur[A != 0].max()
        score = np.array([110.0 + f(mn, mx, c, a) for c, a in zip(cur, A)])
        score[~fit] = -np.inf
        order = np.lexsort((snap.node_name_rank, -score))
        w = order[0]
        mismatches += int(w != res.task_node[t])
        gaps.append((score[w] - score[order[1]]) / np.spacing(score[w]))
        idle[:, w] -= req
    return np.array(gaps), mismatches


def node_summands(snap: abi.Snapshot, r: int) -> np.ndarray:
    """Allocatable - foreign of the Ready nodes in index order: the summands of total_resource[r]."""
    v = snap.node_allocatable[r].copy()
    if snap.node_foreign is not None:
        v = v - snap.node_foreign[r]
    return v[(snap.node_flags & abi.NODE_READY) != 0]


def queue_summands(snap: abi.Snapshot, q: int, r: int, field: str) -> np.ndarray:
    """The task requests the oracle adds into queue q's `field` ("request" | "allocated" | "allocated_np"), in its
    order (job, podset, task = the task index order)."""
    allocated = (snap.task_status & (abi.POD_ALLOCATED | abi.POD_BOUND | abi.POD_BINDING | abi.POD_RUNNING)) != 0
    pending = snap.task_status == abi.POD_PENDING
    t_job = np.repeat(np.arange(snap.n_jobs), np.diff(snap.podset_task_begin[snap.job_podset_begin]))
    under = np.zeros(snap.n_jobs, dtype=bool)
    for j in range(snap.n_jobs):
        a = int(snap.job_queue[j])
        while a >= 0 and a != q:
            a = int(snap.queue_parent[a])
        under[j] = a == q
    keep = under[t_job] & (allocated | pending)
    if field != "request":
        keep &= allocated
    if field == "allocated_np":
        keep &= (snap.job_flags[t_job] & abi.JOB_PREEMPTIBLE) == 0
    return snap.task_req[keep, r]


def sequential(v) -> float:
    acc = 0.0
    for x in np.asarray(v, dtype=np.float64).tolist():
        acc += x
    return acc


def exact(v) -> Fraction:
    return sum((Fraction(x) for x in np.asarray(v, dtype=np.float64).tolist()), Fraction(0))


def sequential_bound(v) -> Fraction:
    """(n-1) * u * sum|v|: the worst-case error of a sequential sum of n terms (Higham, Accuracy and Stability of
    Numerical Algorithms, eq. 4.4, to first order)."""
    v = np.asarray(v, dtype=np.float64)
    return max(len(v) - 1, 0) * Fraction(U) * exact(np.abs(v))


def pairwise(v) -> float:
    v = [float(x) for x in np.asarray(v, dtype=np.float64)]
    while len(v) > 1:
        v = [v[i] + v[i + 1] if i + 1 < len(v) else v[i] for i in range(0, len(v), 2)]
    return v[0] if v else 0.0


def kernel_order_total(snap: abi.Snapshot, r: int, n_sms: int = H100_SMS, block_order=None) -> float:
    """k_node_totals' parallel order: grid-stride thread sums, shuffle-down warp tree, warps of a block in sequence,
    then one atomicAdd per block (in `block_order`, default ascending block index)."""
    N, threads = snap.n_nodes, 256
    blocks = min(n_sms * 4, (N + threads - 1) // threads)
    v = snap.node_allocatable[r].copy()
    if snap.node_foreign is not None:
        v = v - snap.node_foreign[r]
    v[(snap.node_flags & abi.NODE_READY) == 0] = 0.0     # skipped nodes add nothing (+0.0 leaves any sum unchanged)
    stride = blocks * threads
    acc = np.zeros(stride)
    for k in range(0, N, stride):
        chunk = v[k:k + stride]
        acc[:len(chunk)] = acc[:len(chunk)] + chunk
    lanes = acc.reshape(blocks, threads // 32, 32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes.copy()
        lanes[:, :, :32 - o] = lanes[:, :, :32 - o] + lanes[:, :, o:]
    per_block = [sequential(lanes[b, :, 0]) for b in range(blocks)]
    order = range(blocks) if block_order is None else block_order
    total = 0.0
    for b in order:
        total += per_block[b]
    return total


def set_resource_share(total, k, deserved, limit, oqw, request, usage, priority, creation, uid_rank, fair):
    """resource_division.go:26-357 for one sibling group and one resource, in k_fair_share's operations; returns
    (fair shares, paths) where paths counts the floor gifts that left a remainder and the remainder-loop gifts below
    one unit."""
    n = len(deserved)
    fair = [float(x) for x in fair]
    rr = [None] * n
    paths = {"floor_with_remainder": 0, "fractional_remainder_gift": 0}

    def requestable(q):
        return request[q] if limit[q] == -1.0 else min(limit[q], request[q])

    def satisfied(q):
        return request[q] <= fair[q] or (limit[q] != -1.0 and limit[q] <= fair[q])

    def remaining_requested(q):
        r_ = requestable(q)
        return 0.0 if r_ < fair[q] else r_ - fair[q]

    remaining = total
    for q in range(n):
        d = total if deserved[q] == -1.0 else deserved[q]
        amount = min(d, requestable(q))
        fair[q] += amount
        remaining -= amount
    if not remaining > 0:
        return fair, paths
    prios = sorted(set(int(p) for p in priority), reverse=True)
    for p in prios:
        members = [q for q in range(n) if priority[q] == p]
        while True:
            another = False
            round_amount = remaining
            total_w = 0.0
            for q in members:
                if remaining_requested(q) > 0:
                    total_w += oqw[q]
            w, wsum = [0.0] * n, 0.0
            if total_w != 0:
                for q in members:
                    if satisfied(q):
                        continue
                    nw = oqw[q] / total_w
                    sw = max(0.0, nw + k * (nw - (usage[q] if usage is not None else 0.0)))
                    w[q] = sw
                    wsum += sw
            if wsum == 0:
                break
            for q in members:
                if remaining == 0:
                    break
                if satisfied(q):
                    continue
                requested = remaining_requested(q)
                if oqw[q] == 0:
                    continue
                fs = round_amount * (w[q] / wsum)
                give = 0.0
                if requested <= fs:
                    give = requested
                    rr[q] = None
                else:
                    rf = float(np.floor(fs))
                    if rf > 0:
                        give = rf
                    if fs - give > 0:
                        rr[q] = fs - give
                        paths["floor_with_remainder"] += 1
                if give == 0:
                    continue
                fair[q] += give
                remaining -= give
                another = another or requested < fs
            if not another or remaining == 0:
                break
    for p in prios:
        if remaining <= 0:
            break
        members = [q for q in range(n) if priority[q] == p]
        while remaining != 0:
            cand = [q for q in members if rr[q] is not None]
            if not cand:
                break
            best = min(cand, key=lambda q: (-rr[q], creation[q], uid_rank[q]))
            rr[best] = None
            give = min(1.0, remaining)
            if 0 < give < 1:
                paths["fractional_remainder_gift"] += 1
            fair[best] += give
            remaining -= give
    return fair, paths


def fair_share_paths(snap: abi.Snapshot, k: float, tables: abi.Result):
    """Restates the whole hierarchy (proportion.go:403-423) from an engine's / the oracle's open-session tables and
    returns (fair shares [3, Q], summed paths)."""
    Q = snap.n_queues
    fair = np.zeros((3, Q))
    total_paths = {"floor_with_remainder": 0, "fractional_remainder_gift": 0}

    def level(parent_total, group, r):
        res, paths = set_resource_share(
            parent_total, k, [snap.queue_deserved[r, q] for q in group], [snap.queue_limit[r, q] for q in group],
            [snap.queue_oqw[r, q] for q in group], [tables.queue_request[r, q] for q in group],
            None if snap.queue_usage is None else [snap.queue_usage[r, q] for q in group],
            [snap.queue_priority[q] for q in group], [snap.queue_creation[q] for q in group],
            [snap.queue_uid_rank[q] for q in group], [0.0] * len(group))
        for key in paths:
            total_paths[key] += paths[key]
        for q, f in zip(group, res):
            fair[r, q] = f
            children = [c for c in range(Q) if snap.queue_parent[c] == q]
            if children:
                level(f, children, r)

    top = [q for q in range(Q) if snap.queue_parent[q] < 0]
    for r in range(3):
        level(tables.total_resource[r], top, r)
    return fair, total_paths
