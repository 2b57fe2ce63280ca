"""Host-only check of the launch transport's host side (csrc/kai_host_seq.cuh): packing of a decision record into the
kernel parameter block (folded node deltas, flush launches), the merge of several GPUs' candidate lists with the cut
rule applied across ranks — the N > 1 logic that otherwise needs several GPUs — and the reading of single-row and
min-max answer lines under their 64-bit sequence numbers.  Compiled with nvcc as host code."""
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_record_packing_list_merge_and_answer_lines():
    src = os.path.join(ROOT, "tests", "native", "launch_host_check.cu")
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "check")
        subprocess.check_call(["nvcc", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-x", "cu", "-o", exe, src],
                              stdout=subprocess.DEVNULL)
        out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("OK")
