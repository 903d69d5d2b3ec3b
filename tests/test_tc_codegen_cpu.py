"""Codegen guard for the stride-1 tensor-core conv (no GPU needed: nvcc cross-compiles for sm_90a).

ptxas serializes every wgmma of a kernel (one MMA in flight per warpgroup) when it cannot keep the accumulators in a
pipeline: a function call anywhere in the kernel (C7510), too few registers (C7511), or MMA widths chosen at run time.
It says so only as an info message, so this test compiles conv1d_tc.cu with -Xptxas -v and fails on any such message
and on any spill in a conv1d_tc_kernel instantiation."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parallelwavegan_b200", "csrc")


def _nvcc():
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.isfile(cand) and os.access(cand, os.X_OK) else None


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("tc_codegen") / "conv1d_tc.o")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "conv1d_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def _conv_kernel_properties(log):
    """{mangled conv1d_tc_kernel name: (stack, spill stores, spill loads)}"""
    out = {}
    for m in re.finditer(r"Function properties for (\S*conv1d_tc_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                         r"stores, (\d+) bytes spill loads", log):
        out[m.group(1)] = tuple(int(g) for g in m.group(2, 3, 4))
    return out


def test_conv1d_tc_wgmma_not_serialized(ptxas_log):
    assert _conv_kernel_properties(ptxas_log), "no conv1d_tc_kernel in the ptxas report"
    bad = [line for line in ptxas_log.splitlines()
           if "conv1d_tc_kernel" in line and re.search(r"\(C75\d\d\)|serialized", line)]
    assert not bad, "\n".join(bad[:10])


def test_conv1d_tc_no_spills(ptxas_log):
    props = _conv_kernel_properties(ptxas_log)
    # one instantiation per tile shape the planner produces: MT = 1 at 1..8 and MT = 2 at 1..4 16-column blocks
    assert len(props) == 12, sorted(props)
    spilling = {k: v for k, v in props.items() if v[1] or v[2]}
    assert not spilling, spilling
