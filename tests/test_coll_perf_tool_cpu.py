"""The perf tool's flag validation, checked without a GPU: every conflict between modes, dtypes and the rank count is refused once, with
exit status 1, before any communicator exists. On a machine without a GPU a refusal that came later would fail in the library instead."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERF = os.path.join(ROOT, "build", "b200coll_perf")


@pytest.fixture(scope="module")
def perf(coll_lib):
    if not os.path.exists(PERF):
        subprocess.run(["make", "-C", os.path.join(ROOT, "coll"), "../build/b200coll_perf"], check=True, capture_output=True)
    return PERF


@pytest.mark.parametrize("args, message", [
    (["--combine", "2", "--op", "all_reduce"], "--combine K takes --op alltoall"),
    (["--combine", "2", "--op", "alltoall", "--quantize", "e4m3:128"], "--combine K takes --op alltoall"),
    (["--route", "8:2", "--op", "alltoall", "--devs", "0,0,0"], "--route E:K takes --op alltoall"),             # E not a multiple of the ranks
    (["--route", "16:4", "--op", "alltoall", "--quantize", "e4m3:128", "--row-len", "192"], "--route E:K takes --op alltoall"),
    (["--quantize", "e4m3:128", "--op", "broadcast"], "--quantize takes --op all_gather"),
    (["--block-scale", "1x128", "--op", "alltoall"], "--block-scale takes --op all_gather, reduce_scatter or all_reduce"),
    (["--op", "sendrecv", "--out-dtype", "float"], "sendrecv moves opaque bytes"),
    (["--op", "hypercube", "--devs", "0,0,0"], "hypercube needs a power-of-two number of ranks"),
])
def test_refused_before_any_communicator(perf, args, message):
    r = subprocess.run([perf, *args], capture_output=True, text=True, timeout=60)
    assert r.returncode == 1, (args, r.returncode, r.stderr)
    assert r.stderr.count(message) == 1 and r.stdout == "", (args, r.stdout, r.stderr)
