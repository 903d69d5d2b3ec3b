"""Codegen guard and plan of the conv-split fused ResBlock pair (rb_pair_split_kernel, csrc/resblock_tc.cu); no GPU needed.

Each consumer warpgroup of the split kernel keeps 64 accumulator registers and its wgmma groups in flight, which holds
only when ptxas neither serializes the wgmma nor spills: compile the file for sm_90a with -Xptxas -v and fail on either
in an rb_pair_split_kernel instantiation.  The plan (which kernel a pair runs, its tile and its two weight rings) is host
code and is checked through the library."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parallelwavegan_b200", "csrc")
V1 = [(C_, k, d) for C_ in (32, 64) for k in (3, 7, 11) for d in (1, 3, 5)]


def _nvcc():
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.isfile(cand) and os.access(cand, os.X_OK) else None


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("rb_split_codegen") / "resblock_tc.o")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "resblock_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def _split_properties(log):
    """{mangled rb_pair_split_kernel name: (stack, spill stores, spill loads)}"""
    out = {}
    for m in re.finditer(r"Function properties for (\S*rb_pair_split_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                         r"spill stores, (\d+) bytes spill loads", log):
        out[m.group(1)] = tuple(int(g) for g in m.group(2, 3, 4))
    return out


def test_split_kernel_wgmma_not_serialized(ptxas_log):
    assert _split_properties(ptxas_log), "no rb_pair_split_kernel in the ptxas report"
    bad = [line for line in ptxas_log.splitlines() if re.search(r"\(C75\d\d\)|serialized", line)]
    assert not bad, "\n".join(bad[:10])


def test_split_kernel_no_spills(ptxas_log):
    props = _split_properties(ptxas_log)
    assert len(props) == 2, sorted(props)  # 32 channels (256-row tiles) and 64 channels (128-row tiles)
    spilling = {k: v for k, v in props.items() if any(v)}
    assert not spilling, spilling


@pytest.fixture(scope="module")
def ops():
    import __graft_entry__

    __graft_entry__.build()
    from parallelwavegan_b200 import ops

    return ops


@pytest.fixture
def lockstep():
    """pwgb_debug_set(3, 1) for the duration of a test"""
    from parallelwavegan_b200 import capi

    capi.lib().pwgb_debug_set(3, 1)
    yield
    capi.lib().pwgb_debug_set(3, 0)


@pytest.mark.parametrize("channels,k,d", V1)
def test_v1_pairs_run_split(ops, channels, k, d):
    t = 102400 if channels == 32 else 51200
    plan = ops.resblock_pair_plan(channels, t, k, d, batch=16)
    tt = 256 if channels == 32 else 128
    assert plan["variant"] == "split", plan
    assert plan["TT"] == tt and plan["M2"] == (tt - (k - 1)) // 4 * 4, plan
    # two weight rings of at least four stages each
    assert plan["nb"] % 2 == 0 and plan["nb"] >= 8 and plan["nb"] <= 24, plan
    assert plan["na"] >= 1 and plan["ns"] >= 2, plan


@pytest.mark.parametrize("channels,k,d", [(32, 11, 5), (64, 11, 5), (64, 3, 1)])
def test_debug_switch_forces_lockstep(ops, lockstep, channels, k, d):
    t = 102400 if channels == 32 else 51200
    plan = ops.resblock_pair_plan(channels, t, k, d, batch=16)
    assert plan["variant"] == "lockstep", plan
    assert plan["TT"] == (256 if channels == 32 else 128), plan


def test_debug_switch_is_restored(ops):
    assert ops.resblock_pair_plan(64, 51200, 11, 5, batch=16)["variant"] == "split"


def test_wide_dilation_falls_back_to_lockstep(ops):
    """a conv1 halo whose operand buffers leave no room for two rings of four stages still takes the fused path"""
    plan = ops.resblock_pair_plan(64, 51200, 11, 10, batch=16)
    assert plan is not None and plan["variant"] == "lockstep", plan


def test_variant_query_declines_unsupported(ops):
    from parallelwavegan_b200 import capi

    d = capi.ResBlockDesc(batch=1, channels=128, t=1024, kernel=3, dilation=1, slope=0.1, out_scale=1.0, accumulate=0)
    assert capi.lib().pwgb_resblock_pair_variant(C.byref(d)) == 0
