"""Host build of the scanners' node scoring (node_key / repeat_row / binpack_score / better in csrc/kai_action.cuh)
against the oracle.

The solver answers small restricted simulation sweeps on the host with the same source the GPU scanners run, so the
host build has to reproduce the oracle's NodeOrderFn sum (oracle/kai_oracle.cpp, session_plugins.go:427-437) bit for
bit: value regime (c)'s edges (ulp-close scores, exact ties broken by name rank, mn == mx, mx == 0, overall == 0) and
the nominated-node, best-effort and CPU-only-node terms.  The scanners' same-node repeat analysis (repeat_row) scores a
winning row after k further placements; it has to match the oracle's scoring of the row after k sequential
subtractions, in Idle and Releasing mode.  Compiled with nvcc as host code; no GPU needed."""
import math
import os
import random
import shutil
import subprocess
import tempfile

import pytest

from oracle_lib import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU, MEM, GPU = 0, 1, 2
BINPACK, SPREAD = 0, 1
NOT_CPU_ONLY = 2
RANK_NONE = 0xFFFFFF
R = 4


def _run(lines):
    src = os.path.join(ROOT, "tests", "native", "host_score_check.cu")
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "check")
        subprocess.check_call(["nvcc", "-O1", "-std=c++17", "-Xcompiler", "-ffp-contract=off", "-gencode",
                               "arch=compute_90a,code=sm_90a", "-x", "cu", "-o", exe, src], stdout=subprocess.DEVNULL)
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    res = out.stdout.splitlines()
    assert res[-1] == "OK", out.stdout
    return res[:-1]


def _h(x: float) -> str:
    return float(x).hex()


def _empty(req):  # best-effort pod: the engine's rule for a request the oracle calls empty
    e = not (req[GPU] > 0.01) and not (req[CPU] >= 10) and not (req[MEM] >= 10.0 * 1024 * 1024)
    return e and all(not (req[r] >= 10) for r in range(3, R))


def _fits(req, I, L=None):
    """The request fits on Idle (+ Releasing when L is given)."""
    for r in range(R):
        avail = I[r] + L[r] if L is not None else I[r]
        if r >= 3:
            if req[r] != 0 and req[r] > avail:
                return False
        elif req[r] > avail:
            return False
    return True


def _oracle_key(c):
    """(fits, fit_i, score) in the oracle's order (kai_oracle.cpp: fits / is_task_allocatable / the NodeOrderFn sum)."""
    req, I, L = c["req"], c["I"], c["L"]
    if not _fits(req, I, L):
        return 0, 0, 0.0
    fit_i = _fits(req, I)
    res = c["res"]
    score = 0.0
    score += 100.0 if (_empty(req) or fit_i) else 0.0
    score += 0.0
    cpu_only = not (c["nflags"] & NOT_CPU_ONLY) and c["a_gpu"] <= 0
    score += 10.0 if (not c["gpu_task"] and cpu_only) else 0.0
    score += 1000000.0 if c["nominated"] == c["n"] else 0.0
    cur = I[res] + L[res]
    overall = c["a_gpu"] if res == GPU else c["a_cpu"]
    if c["strategy"] == BINPACK:
        score += lib().kai_oracle_binpack_score(c["mn"], c["mx"], cur, overall)
    else:
        score += lib().kai_oracle_spread_score(cur, float(int(c["gpu_count"])) if res == GPU else overall)
    return 1, int(fit_i), score


def _cases():
    rnd = random.Random(7)
    out = []
    base_cpu = 1.3e4 + 1 / 3  # regime (c): non-round CPU-only scores

    def case(**kw):
        c = dict(strategy=BINPACK, nominated=-1, n=5, mn=0.0, mx=0.0, a_gpu=0.0, a_cpu=2.1e4 + 0.7, gpu_count=0.0,
                 nflags=0, req=[1000.0, 1e9, 0.0, 0.0], I=[base_cpu, 3e10, 0.0, 110.0], L=[0.0, 0.0, 0.0, 0.0])
        c.update(kw)
        c["res"] = GPU if c["req"][GPU] > 0 else CPU
        c["gpu_task"] = int(c["req"][GPU] > 0)
        out.append(c)

    # CPU-only nodes, binpack over ulp-close idle CPU values
    cur = base_cpu
    for k in range(6):
        nxt = math.nextafter(cur, math.inf)
        case(mn=base_cpu, mx=math.nextafter(base_cpu, math.inf) + 3e-12, I=[nxt, 3e10, 0.0, 110.0])
        cur = nxt
    case(mn=base_cpu, mx=base_cpu)                      # mn == mx
    case(mn=base_cpu, mx=0.0)                           # mx == 0
    case(mn=1.0, mx=2e4, a_cpu=0.0)                     # overall == 0
    case(mn=7.25, mx=2.1e4 + 0.7, nominated=5)          # the nominated node
    case(mn=7.25, mx=2.1e4 + 0.7, nflags=NOT_CPU_ONLY)  # not a CPU-only node
    case(req=[5.0, 1024.0, 0.0, 0.0], I=[3.0, 10.0, 0.0, 0.0], L=[4.0, 0.0, 0.0, 0.0], mn=1.0, mx=9.5)  # best effort
    case(req=[20.0, 1e9, 0.0, 0.0], I=[10.0, 3e10, 0.0, 0.0], L=[15.0, 0.0, 0.0, 0.0], mn=1.0, mx=30.0)  # fits on releasing
    case(req=[20.0, 1e9, 0.0, 0.0], I=[10.0, 3e10, 0.0, 0.0], L=[5.0, 0.0, 0.0, 0.0], mn=1.0, mx=30.0)   # does not fit
    case(req=[20.0, 1e9, 0.0, 5.0], I=[40.0, 3e10, 0.0, 4.0], L=[0.0, 0.0, 0.0, 0.5], mn=1.0, mx=30.0)   # scalar short
    # GPU nodes: binpack and spread, whole and odd GPU counts
    for k in range(40):
        gi = float(rnd.randint(0, 8))
        gl = float(rnd.randint(0, 2))
        case(req=[1000.0 + rnd.random(), 1e9 + rnd.randint(0, 999), float(rnd.randint(1, 4)), 0.0],
             I=[2e4 + rnd.random() * 1e4, 3e12 + rnd.randint(0, 10**6), gi, 110.0], L=[rnd.random() * 10, 0.0, gl, 0.0],
             a_gpu=8.0, gpu_count=8.0 if k % 3 else 7.0, strategy=SPREAD if k % 4 == 0 else BINPACK,
             mn=float(rnd.randint(0, 3)), mx=float(rnd.randint(3, 10)) if k % 5 else float(rnd.randint(0, 3)),
             nominated=5 if k % 7 == 0 else -1, nflags=NOT_CPU_ONLY if k % 2 else 0)
    # CPU task on GPU nodes and on CPU-only nodes, spread on CPU (count = allocatable CPU)
    for k in range(20):
        case(strategy=SPREAD if k % 2 else BINPACK, a_gpu=0.0 if k % 3 else 4.0, mn=rnd.random() * 1e4,
             mx=1e4 + rnd.random() * 1e4, I=[rnd.random() * 2e4 + 1000.0, 3e10, 0.0, 110.0], L=[rnd.random(), 0.0, 0.0, 0.0])
    return out


def _oracle_repeat(c):
    """(to_idle, repeat ok, fits, fit_i, score) of the row after c["k"] placements: the mode is decided on the row before
    them (common/allocate.go:165-174), each placement subtracts the request (node_info.go:457-493), the oracle scores the
    result, and placement k may repeat a winner of score c["win"] if it fits, in the same mode, at a score not below it."""
    req = c["req"]
    best_effort = _empty(req)
    to_idle = not c["pipeline_only"] and (best_effort or _fits(req, c["I"]))
    I, L = list(c["I"]), list(c["L"])
    for _ in range(c["k"]):
        for r in range(R):
            if to_idle:
                I[r] -= req[r]
            else:
                L[r] -= req[r]
    fits, fit_i, score = _oracle_key(dict(c, I=I, L=L))
    same_mode = (not c["pipeline_only"] and (best_effort or fit_i)) == to_idle
    return int(to_idle), int(bool(fits) and same_mode and score >= c["win"]), fits, fit_i, score


def _repeat_cases():
    """Rows that take several placements of one request, k = 0..10 each: Idle and Releasing mode, an Idle row whose
    Idle runs out first (the mode would change, also while the binpack score keeps rising), pipeline-only and best-effort pods, a scalar resource, binpack (the score
    rises as the row fills) and spread (it falls) on CPU-only and GPU rows.  The winning score is the row's own score
    before the placements, or the next double above it."""
    rnd = random.Random(11)
    cpu_req = [1000.0 + 1 / 3, 1e9, 0.0, 0.0]
    rows = [
        dict(req=cpu_req, I=[7.3e3 + 1 / 7, 3e10, 0.0, 110.0], mn=1.3e3, mx=2.1e4 + 0.7),                 # Idle
        dict(req=cpu_req, I=[7.3e3 + 1 / 7, 3e10, 0.0, 110.0], mn=1.3e3, mx=2.1e4 + 0.7, strategy=SPREAD),
        dict(req=cpu_req, I=[500.25, 3e10, 0.0, 110.0], L=[8.2e3 + 1 / 3, 0.0, 0.0, 0.0], mn=1.0, mx=9e3),  # Releasing
        dict(req=cpu_req, I=[3.2e3 + 1 / 9, 3e10, 0.0, 110.0], L=[5e3, 0.0, 0.0, 0.0], mn=1.0, mx=9e3),     # Idle runs out
        dict(req=cpu_req, I=[3.2e3 + 1 / 9, 3e10, 0.0, 110.0], L=[5e3, 0.0, 0.0, 0.0], mn=9e3, mx=9e3 + 1),  # score still rises
        dict(req=cpu_req, I=[9.1e3 + 0.1, 3e10, 0.0, 110.0], mn=1.0, mx=9.2e3, pipeline_only=1),
        dict(req=[5.0, 1024.0, 0.0, 0.0], I=[30.0, 1e4, 0.0, 0.0], L=[7.5, 0.0, 0.0, 0.0], mn=1.0, mx=40.0),  # best effort
        dict(req=[1000.0, 1e9, 0.0, 5.0], I=[2e4, 3e10, 0.0, 40.0], L=[0.0, 0.0, 0.0, 0.5], mn=1.0, mx=3e4),  # scalar
        dict(req=[1000.5, 1e9 + 7, 1.0, 0.0], I=[2.4e4 + 0.3, 3e12, 6.0, 110.0], L=[3.7, 0.0, 2.0, 0.0],
             a_gpu=8.0, gpu_count=8.0, mn=0.0, mx=8.0, nflags=NOT_CPU_ONLY),
        dict(req=[1000.5, 1e9 + 7, 1.0, 0.0], I=[2.4e4 + 0.3, 3e12, 6.0, 110.0], L=[3.7, 0.0, 2.0, 0.0],
             a_gpu=8.0, gpu_count=7.0, strategy=SPREAD, nominated=5),
        dict(req=[1000.5, 1e9 + 7, 2.0, 0.0], I=[2.4e4 + 0.3, 3e12, 0.0, 110.0], L=[3.7, 0.0, 7.0, 0.0],
             a_gpu=8.0, gpu_count=8.0, mn=1.0, mx=7.0),                                                    # GPU Releasing
    ]
    for k in range(6):
        rows.append(dict(req=[1000.0 + rnd.random(), 1e9 + rnd.randint(0, 999), float(rnd.randint(1, 2)), 0.0],
                         I=[2e4 + rnd.random() * 1e4, 3e12 + rnd.randint(0, 10**6), float(rnd.randint(0, 8)), 110.0],
                         L=[rnd.random() * 10, 0.0, float(rnd.randint(0, 4)), 0.0], a_gpu=8.0, gpu_count=8.0,
                         strategy=SPREAD if k % 2 else BINPACK, mn=float(rnd.randint(0, 3)), mx=float(rnd.randint(3, 10))))
    out = []
    for row in rows:
        c = dict(strategy=BINPACK, nominated=-1, n=5, mn=0.0, mx=0.0, a_gpu=0.0, a_cpu=2.1e4 + 0.7, gpu_count=0.0,
                 nflags=0, L=[0.0, 0.0, 0.0, 0.0], pipeline_only=0)
        c.update(row)
        c["res"] = GPU if c["req"][GPU] > 0 else CPU
        c["gpu_task"] = int(c["req"][GPU] > 0)
        _, _, _, _, win = _oracle_repeat(dict(c, k=0, win=0.0))
        for k in range(11):
            out.append(dict(c, k=k, win=win))
            out.append(dict(c, k=k, win=math.nextafter(win, math.inf)))
    return out


def _key_fields(c):
    vals = [c["strategy"], c["res"], c["gpu_task"], int(_empty(c["req"])), c["nominated"], c["n"], _h(c["mn"]), _h(c["mx"]),
            _h(c["a_gpu"]), _h(c["a_cpu"]), _h(c["gpu_count"]), c["nflags"]]
    vals += [_h(v) for v in c["req"] + c["I"] + c["L"]]
    return "%d " % R + " ".join(str(v) for v in vals)


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_host_node_scoring_matches_the_oracle():
    cases = _cases()
    lines = ["K " + _key_fields(c) for c in cases]
    # binpack_score edges and ulp-close currents, against the oracle's getScoreOfCurrentNode
    pcases = [(0.0, 0.0, 0.0, 8.0), (3.0, 3.0, 3.0, 8.0), (1.0, 5.0, 2.0, 0.0), (0.0, 8.0, 3.0, 8.0)]
    x = 1.3e4 + 1 / 3
    for k in range(8):
        pcases.append((1.3e4 + 1 / 3, math.nextafter(1.3e4 + 1 / 3, math.inf) + 1e-11, x, 2.1e4 + 0.7))
        x = math.nextafter(x, math.inf)
    lines += ["P " + " ".join(_h(v) for v in pc) for pc in pcases]
    # argmax order: score desc, then name rank asc; an empty slot never wins
    s = 109.0 + 1 / 3
    bcases = [(s, 4, s, 9), (s, 9, s, 4), (s, 4, s, 4), (math.nextafter(s, 0), 1, s, 2), (s, 2, math.nextafter(s, 0), 1),
              (s, RANK_NONE, -1.0, RANK_NONE), (-1.0, 3, s, RANK_NONE), (s, 3, s, RANK_NONE), (s, RANK_NONE, s, 3)]
    lines += ["B %s %d %s %d" % (_h(a), ra, _h(b), rb) for a, ra, b, rb in bcases]
    # the repeat analysis: the row after k placements, scored
    rcases = _repeat_cases()
    lines += ["A %s %d %d %s" % (_key_fields(c), c["pipeline_only"], c["k"], _h(c["win"])) for c in rcases]
    got = _run(lines)
    assert len(got) == len(lines)
    n_fit, scores = 0, set()
    for c, g in zip(cases, got):
        f = g.split()
        fits, fit_i, score = _oracle_key(c)
        assert (int(f[1]), int(f[2])) == (fits, fit_i), (c, g)
        if fits:
            n_fit += 1
            assert float.fromhex(f[3]).hex() == score.hex(), (c, g, score.hex())
            scores.add(score)
    assert n_fit > 40 and len(scores) > 20  # the cases reach many distinct scores, not one path
    for pc, g in zip(pcases, got[len(cases):]):
        assert float.fromhex(g.split()[1]).hex() == _h(lib().kai_oracle_binpack_score(*pc)), (pc, g)
    for (a, ra, b, rb), g in zip(bcases, got[len(cases) + len(pcases):]):
        want = ra != RANK_NONE and (rb == RANK_NONE or a > b or (a == b and ra < rb))
        assert g == "B %d" % int(want), ((a, ra, b, rb), g)
    seen = set()
    for c, g in zip(rcases, got[len(cases) + len(pcases) + len(bcases):]):
        f = g.split()
        to_idle, ok, fits, fit_i, score = _oracle_repeat(c)
        assert f[0] == "A" and tuple(int(x) for x in f[1:5]) == (to_idle, ok, fits, fit_i), (c, g)
        if fits:
            assert float.fromhex(f[5]).hex() == score.hex(), (c, g, score.hex())
        seen.add((to_idle, ok, fits, fit_i, c["k"] > 0))
    # both modes, repeats taken and refused, rows that stop fitting and rows that leave Idle while still fitting
    assert {(1, 1, 1, 1, True), (0, 1, 1, 0, True), (1, 0, 0, 0, True), (0, 0, 0, 0, True), (1, 0, 1, 0, True)} <= seen, seen
