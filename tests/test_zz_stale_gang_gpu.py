"""stalegangeviction with a grace period on the engine (GPU): the reference's own table
(actions/stalegangeviction/stalegangeviction_test.go, grace period 60 s, per-job staleness timestamps) through the C ABI,
against the oracle and against the table's expectations; plus the grace-period variations on a synthetic cluster.

Kept in its own late-sorting file: `job_stale_since_s` (ABI v6) was added after the round's last GPU minutes.
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dsl  # noqa: E402
from fixtures import action_cases, case_config  # noqa: E402
from test_engine_gpu import assert_same, run_both  # noqa: E402

from kai_scheduler_b200 import abi  # noqa: E402

pytestmark = pytest.mark.gpu

STALE = action_cases(["stalegangeviction__"], single_action="stalegangeviction")


@pytest.mark.parametrize("cid,case", STALE, ids=[c[0] for c in STALE])
def test_stale_gang_eviction_table_gpu(cid, case):
    snap, meta = dsl.build_snapshot(case["topology"])
    re_, ro = run_both(snap, action="stalegangeviction", cfg=case_config(case))
    assert_same(re_, ro)
    assert re_.pods_evicted == ro.pods_evicted
    errs = dsl.check_expectations(case["topology"], meta, re_, snap)
    assert not errs, f"{case['source']} #{case['index']} {case['name']}: {errs}"


@pytest.mark.parametrize("grace", [-1, 0, 30, 60, 3600])
def test_grace_period_variations_gpu(grace):
    """Gangs knocked below minAvailable at different instants: only those stale for at least the grace period go; a gang
    without a timestamp counts as stale since `now` (see tests/test_stale_gang_units.py for the expected counts)."""
    from test_stale_gang_units import stale_cluster
    snap, meta = dsl.build_snapshot(stale_cluster())
    re_, ro = run_both(snap, action="stalegangeviction", cfg=abi.make_config(staleness_grace_period_s=grace))
    assert_same(re_, ro)
    assert re_.pods_evicted == ro.pods_evicted
    if grace < 0:
        assert re_.pods_evicted == 0


@pytest.mark.parametrize("cid,case", STALE, ids=[c[0] for c in STALE])
def test_stale_gang_eviction_through_cpp_shim(cid, case):
    """The same table through the C++ mirror of the Go shim (host/): `stalegangeviction` from the Action registry, the
    session replays the evictions."""
    import subprocess
    import tempfile

    import numpy as np
    import test_host_cpp as hc
    hc._build()
    snap, meta = dsl.build_snapshot(case["topology"])
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "case.txt")
        hc.write_case(path, snap, meta, case["actions"], case["topology"], cfg=case["config"])
        out = subprocess.run([hc.BIN, path], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = [l.split() for l in out.stdout.strip().split("\n")]
    by_name = {l[0]: l for l in lines if l[0] != "cache"}
    res = hc._Res()
    res.task_status = np.array([int(by_name[n][1]) for n in meta["task_names"]], dtype=np.int32)
    nidx = {n: i for i, n in enumerate(meta["node_names"])}
    res.task_node = np.array([nidx.get(by_name[n][2], -1) for n in meta["task_names"]], dtype=np.int32)
    res.node_idle = res.node_releasing = None
    errs = dsl.check_expectations(case["topology"], meta, res, snap)
    assert not errs, f"{case['source']} #{case['index']} {case['name']}: {errs}"
