"""Codegen guard and plan rule of the fused ResBlock conv pair (rb_pair_split_kernel, csrc/resblock_tc.cu); no GPU needed.

Each consumer warpgroup of the kernel keeps 64 accumulator registers and its wgmma groups in flight, which holds only
when ptxas neither serializes the wgmma nor spills, and ptxas reports serialization only as an info message (as for the
stride-1 conv, tests/test_tc_codegen_cpu.py): compile the file for sm_90a with -Xptxas -v and fail on any such message
and on any stack or spill in an rb_pair_split_kernel instantiation.  The plan rule (which pairs take the fused kernel,
its tile and its two weight rings) is host code and is checked through the library."""
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
    obj = str(tmp_path_factory.mktemp("rb_codegen") / "resblock_tc.o")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-I", CSRC, "-Xptxas", "-v", "-c", os.path.join(CSRC, "resblock_tc.cu"), "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def _kernel_properties(log):
    """{mangled rb_pair_split_kernel name: (stack, spill stores, spill loads)}"""
    out = {}
    for m in re.finditer(r"Function properties for (\S*rb_pair_split_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                         r"spill stores, (\d+) bytes spill loads", log):
        out[m.group(1)] = tuple(int(g) for g in m.group(2, 3, 4))
    return out


def test_split_kernel_wgmma_not_serialized(ptxas_log):
    assert _kernel_properties(ptxas_log), "no rb_pair_split_kernel in the ptxas report"
    bad = [line for line in ptxas_log.splitlines() if re.search(r"\(C75\d\d\)|serialized", line)]
    assert not bad, "\n".join(bad[:10])


def test_split_kernel_no_spills(ptxas_log):
    props = _kernel_properties(ptxas_log)
    assert len(props) == 2, sorted(props)  # 32 channels (256-row tiles) and 64 channels (128-row tiles)
    spilling = {k: v for k, v in props.items() if any(v)}
    assert not spilling, spilling


@pytest.fixture(scope="module")
def ops():
    import __graft_entry__

    __graft_entry__.build()
    from parallelwavegan_b200 import ops

    return ops


@pytest.mark.parametrize("channels,t", [(32, 102400), (64, 51200)])
@pytest.mark.parametrize("k,dilations", [(3, (1, 3, 5)), (7, (1, 3, 5)), (11, (1, 3, 5))])
def test_v1_pairs_at_32_and_64_channels_are_fused(ops, channels, t, k, dilations):
    for d in dilations:
        plan = ops.resblock_pair_plan(channels, t, k, d, batch=16)
        assert plan is not None, (channels, k, d)
        # a 256-row (32 channels) or 128-row (64 channels) conv tile minus the conv2 halo, in 16-byte output rows
        tt = 256 if channels == 32 else 128
        assert plan["TT"] == tt and plan["M2"] == (tt - (k - 1)) // 4 * 4, plan
        # two weight rings of at least four stages each
        assert plan["nb"] % 2 == 0 and 8 <= plan["nb"] <= 24, plan
        assert plan["na"] >= 1 and plan["ns"] >= 2, plan


@pytest.mark.parametrize("channels,t", [(128, 25600), (256, 3200), (48, 4096)])
def test_other_channel_counts_keep_two_launches(ops, channels, t):
    assert ops.resblock_pair_plan(channels, t, 3, 1) is None


def test_ragged_length_keeps_two_launches(ops):
    assert ops.resblock_pair_plan(32, 2049, 3, 1) is None
    assert ops.resblock_pair_plan(32, 2052, 3, 1) is not None


def test_wide_halo_keeps_two_launches(ops):
    """a conv1 halo whose operand buffers leave no room for two weight rings of four stages each has no plan"""
    # (channels, k, the first dilation without a plan)
    for channels, k, d in [(64, 11, 6), (64, 7, 11), (64, 3, 31), (32, 11, 9), (32, 7, 15), (32, 3, 43)]:
        t = 102400 if channels == 32 else 51200
        assert ops.resblock_pair_plan(channels, t, k, d - 1, batch=16) is not None, (channels, k, d - 1)
        wider = [dd for dd in range(d, 2 * d) if ops.resblock_pair_plan(channels, t, k, dd, batch=16) is not None]
        assert not wider, (channels, k, wider)
