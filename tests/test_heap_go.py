"""The solver's heap (HeapGo in csrc/kai_solver.cuh) pops in exactly Go container/heap's order.

Every JobsOrder heap (root, queue nodes, leaves) runs HeapGo's sift code on its range of one arena.  The queue-order
comparators are not antisymmetric, so the pop order depends on the exact sift sequence.  tests/native/heap_go_check.cu
drives HeapGo and a plain restatement of container/heap with the same random push / pop / fix sequences under random
non-antisymmetric relations and compares the heap arrays after every step.  Compiled with nvcc as host code; no GPU
needed."""
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_heap_go_matches_container_heap():
    src = os.path.join(ROOT, "tests", "native", "heap_go_check.cu")
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "check")
        subprocess.check_call(["nvcc", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-x", "cu",
                               "-o", exe, src], stdout=subprocess.DEVNULL)
        for seed in range(1, 201):
            out = subprocess.run([exe, str(seed), "3000"], capture_output=True, text=True)
            assert out.returncode == 0 and out.stdout.strip() == "OK", out.stdout + out.stderr
