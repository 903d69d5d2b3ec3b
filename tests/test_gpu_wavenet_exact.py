"""Both WaveNet layer forms against the exact bf16x3 emulation (oracle/bf16x3.py: wavenet_layer, pack_words, gate_bound).

- fused: pwgb_wnstack_layer_forward (one wavenet_fused_kernel per layer on the packed hi / lo residual stream), the
  PWG inference layer;
- two: pwgb_wavenet_layer_forward (two conv1d_tc launches: conv + aux 1x1 into g_ws, then the pre_gate producer and
  the EPI_WAVENET split epilogue), the PWG training layer.

The gate (ex2.approx / div.approx in the fused form, tanhf / __expf in the two-launch form) cannot be emulated bit for
bit, so the end-to-end cases use data on which its output is exactly known, and a derived per-element bound elsewhere:
- launch1: general grid data; g_ws must equal the emulated g (the gate does not enter it);
- zero: c = the conv of x and W_aux = -I, so g == 0 and z == 0: any wrong tap, row, halo, chunk or dropped product of
  the conv makes z != 0, which shows in the skips (lo parts on x, or on the weights, for both cross products);
- sat: W_conv = 0, W_aux = I and c in the gate's exact classes (EXACT_TANH / EXACT_SIGMOID), so z is exactly 0, +-0.5
  or +-1: pins the z image / pre_gate producer, the skip / out contraction, the biases, skips_init, write_x and the
  sqrt(1/2) rounding and hi / lo write of x';
- bound (fused): general grid data with a conv bias; |dev - ref| <= gate_bound per element on skips and x'.
test_gate_readout reads the device gates back first and checks the identities the exact classes rely on.
"""
import ctypes as C
import math
import zlib

import pytest
import torch

from oracle import bf16x3 as E

pytestmark = pytest.mark.gpu

K = 3
V1 = (64, 128, 64, 128)
SHAPES = [V1, (32, 64, 32, 64), (96, 128, 32, 128), (32, 128, 96, 128)]

# name: (form, (R, G, S, A), B, T, dilation, max dilation of the halo (fused), regime, skips_init, write_x)
CASES = {
    # launch 1 of the two-launch form: aux widths, contiguous-tile and window plans, ragged T, many tiles
    "l1_a32_d1": ("two", (64, 128, 64, 32), 2, 515, 1, None, "launch1", False, True),
    "l1_a64_d2": ("two", (64, 128, 64, 64), 2, 257, 2, None, "launch1", False, True),
    "l1_a96_d8": ("two", (64, 128, 64, 96), 1, 1000, 8, None, "launch1", False, True),
    "l1_a128_d64": ("two", (64, 128, 64, 128), 2, 700, 64, None, "launch1", False, True),
    "l1_a96_d128_win": ("two", (64, 128, 64, 96), 1, 1500, 128, None, "launch1", False, True),
    "l1_a96_d256_win": ("two", (64, 128, 64, 96), 1, 1300, 256, None, "launch1", False, True),
    "l1_a96_d512_win": ("two", (64, 128, 64, 96), 1, 2100, 512, None, "launch1", False, True),
    "l1_a96_d512_t100": ("two", (64, 128, 64, 96), 2, 100, 512, None, "launch1", False, True),
    "l1_a32_r32": ("two", (32, 64, 32, 32), 2, 127, 4, None, "launch1", False, True),
    "l1_many_tiles": ("two", (64, 128, 64, 96), 3, 128 * 150, 2, None, "launch1", False, True),
    # two-launch end to end
    "two_zero_x_d1": ("two", V1, 2, 256, 1, None, "zero_x", False, True),
    "two_zero_w_d512": ("two", V1, 1, 1100, 512, None, "zero_w", False, True),
    "two_zero_x_r32": ("two", (32, 64, 32, 64), 2, 129, 8, None, "zero_x", False, True),
    "two_zero_w_r96": ("two", (96, 128, 32, 128), 1, 255, 64, None, "zero_w", False, True),
    "two_sat_v1": ("two", V1, 2, 515, 2, None, "sat", False, True),
    "two_sat_r32": ("two", (32, 64, 32, 64), 2, 4, 1, None, "sat", False, True),
    "two_sat_r96": ("two", (96, 128, 32, 128), 1, 127, 128, None, "sat", False, True),
    "two_sat_s96": ("two", (32, 128, 96, 128), 1, 1, 1, None, "sat", False, True),
    "two_b0": ("two", V1, 0, 256, 1, None, "sat", False, True),
    # fused: zero target over dilations, tight and loose halos, tile edges, ring wraps
    "fz_x_d1": ("fused", V1, 2, 128, 1, 1, "zero_x", True, True),
    "fz_w_d1": ("fused", V1, 2, 129, 1, 1, "zero_w", True, True),
    "fz_x_d2_loose": ("fused", V1, 1, 255, 2, 64, "zero_x", True, True),
    "fz_w_d8": ("fused", V1, 1, 256, 8, 8, "zero_w", True, True),
    "fz_x_d64": ("fused", V1, 1, 257, 64, 64, "zero_x", True, True),
    "fz_w_d128": ("fused", V1, 1, 515, 128, 512, "zero_w", True, True),
    "fz_x_d256": ("fused", V1, 1, 515, 256, 256, "zero_x", True, True),
    "fz_w_d512": ("fused", V1, 1, 1100, 512, 512, "zero_w", True, True),
    "fz_x_d512_t100": ("fused", V1, 2, 100, 512, 512, "zero_x", True, True),
    "fz_x_t1": ("fused", V1, 2, 1, 1, 1, "zero_x", True, True),
    "fz_w_t4": ("fused", V1, 2, 4, 2, 2, "zero_w", True, True),
    "fz_x_r32": ("fused", (32, 64, 32, 64), 2, 127, 4, 4, "zero_x", True, True),
    "fz_w_r96": ("fused", (96, 128, 32, 128), 1, 300, 16, 16, "zero_w", True, True),
    "fz_x_s96": ("fused", (32, 128, 96, 128), 1, 300, 16, 32, "zero_x", True, True),
    "fz_many_tiles": ("fused", V1, 3, 128 * 150, 2, 2, "zero_x", True, True),
    # fused: saturated gate, skips_init both ways, write_x off
    "fs_v1_acc": ("fused", V1, 2, 515, 4, 8, "sat", False, True),
    "fs_v1_init": ("fused", V1, 2, 515, 4, 8, "sat", True, True),
    "fs_v1_nowrite": ("fused", V1, 2, 257, 1, 1, "sat", False, False),
    "fs_r32": ("fused", (32, 64, 32, 64), 2, 128, 1, 1, "sat", False, True),
    "fs_r96": ("fused", (96, 128, 32, 128), 1, 129, 2, 2, "sat", True, True),
    "fs_s96": ("fused", (32, 128, 96, 128), 1, 255, 512, 512, "sat", False, True),
    "fs_many_tiles": ("fused", V1, 3, 128 * 150, 1, 1, "sat", False, True),
    "fs_b0": ("fused", V1, 0, 256, 1, 1, "sat", False, True),
    # fused: bound regime (general data, conv bias)
    "fb_v1_a80": ("fused", (64, 128, 64, 80), 2, 1000, 2, 2, "bound", False, True),
    "fb_v1": ("fused", V1, 2, 1000, 16, 16, "bound", False, True),
    "fb_r32": ("fused", (32, 64, 32, 64), 2, 4000, 1, 1, "bound", False, True),
    "fb_r96": ("fused", (96, 128, 32, 128), 1, 1000, 512, 512, "bound", False, True),
    "fb_s96": ("fused", (32, 128, 96, 128), 1, 1000, 8, 8, "bound", False, True),
}


def case_data(name):
    """The inputs of case ``name`` (CPU tensors, one generator per case)."""
    form, (R, G, S, A), B, T, d, _, regime, _, _ = CASES[name]
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    if regime == "launch1":
        H = G // 2
        x = E.grid_values((B, R, T), gen, 1.0, hmax=1)
        c = E.grid_values((B, A, T), gen, 1.0, hmax=1)
        return dict(x=x, c=c, w_conv=E.grid_values((G, R, K), gen, 2.0 ** -3, hmax=1),
                    b_conv=E.grid_values((G,), gen, 2.0 ** -1, hmax=3), w_aux=E.grid_values((G, A), gen, 2.0 ** -3, hmax=1),
                    w_skip=E.grid_values((S, H), gen, 2.0 ** -3), w_out=E.grid_values((R, H), gen, 2.0 ** -3),
                    b_skip=None, b_out=None, skips=torch.zeros(B, S, T))
    if regime in ("zero_x", "zero_w"):
        return E.zero_target_data(gen, B, R, G, S, T, K, d, lo_on=regime[-1])
    if regime == "sat":
        return E.saturated_data(gen, B, R, G, S, T, form)
    return E.bound_data(gen, B, R, G, S, A, T, K)


def case_emulation(name):
    form, shape, B, T, d, _, regime, skips_init, _ = CASES[name]
    dd = case_data(name)
    gate = None if regime in ("launch1", "bound") else E.gate_table(form)
    emu = E.wavenet_layer(dd["x"], dd["c"], dd["w_conv"], dd["b_conv"], dd["w_aux"], dd["w_skip"], dd["b_skip"], dd["w_out"],
                          dd["b_out"], dilation=d, form=form, gate=gate, skips=dd["skips"], skips_init=skips_init)
    return dd, emu


def _assert_equal(y, ref, what):
    y = y.detach().cpu()
    assert y.shape == ref.shape, (what, tuple(y.shape), tuple(ref.shape))
    if torch.equal(y, ref):
        return
    bad = (y != ref).nonzero()
    dlt = (y.double() - ref.double()).abs()
    raise AssertionError(f"{what}: {bad.shape[0]} of {ref.numel()} elements differ, first at {bad[:4].tolist()}, "
                         f"max |diff| {float(dlt.max()):.3e}")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _tp(T, halo):
    return 2 * halo + (T + 255) // 256 * 256


def run_two(dev, name, dd):
    """pwgb_wavenet_layer_forward with caller-owned g_ws: (g_ws, x', skips) on the CPU"""
    from parallelwavegan_b200 import capi, ops

    form, (R, G, S, A), B, T, d, _, _, _, _ = CASES[name]
    cu = {k: (v.to(dev).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in dd.items()}
    packed, bso = ops.wavenet_packed_weights(cu["w_conv"], cu["w_aux"], cu["w_skip"], cu["w_out"], cu["b_skip"], cu["b_out"], A)
    desc = capi.WaveNetDesc(batch=B, t=T, residual_channels=R, gate_channels=G, skip_channels=S, aux_channels=A, kernel=K,
                            dilation=d)
    L = capi.lib()
    assert L.pwgb_wavenet_supported(C.byref(desc))
    g_ws = torch.full((B, G, T), math.nan, device=dev)
    x_out = torch.full((B, R, T), math.nan, device=dev)
    skips = cu["skips"].clone()
    rc = L.pwgb_wavenet_layer_forward(C.byref(desc), _p(cu["x"]), _p(cu["c"]), _p(packed), _p(cu["b_conv"]), _p(bso),
                                      _p(x_out), _p(skips), _p(g_ws), ops._stream())
    capi.check(rc, "pwgb_wavenet_layer_forward")
    torch.cuda.synchronize()
    return g_ws.cpu(), x_out.cpu(), skips.cpu()


def run_fused(dev, name, dd):
    """pack_c / pack_x / pwgb_wnstack_layer_forward: (input words, output words, skips) on the CPU"""
    from parallelwavegan_b200 import ops

    form, (R, G, S, A), B, T, d, dmax, _, skips_init, write_x = CASES[name]
    cu = {k: (v.to(dev).contiguous() if isinstance(v, torch.Tensor) else v) for k, v in dd.items()}
    assert ops.WnStack.supported(B, T, R, G, S, A, K, dmax)
    st = ops.WnStack(B, T, R, G, S, A, K, dmax, dev)
    st.pack_c(cu["c"])
    st.pack_x(cu["x"])
    words_in = st.x[st.cur].clone()
    packed, bso = ops.wavenet_packed_weights(cu["w_conv"], cu["w_aux"], cu["w_skip"], cu["w_out"], cu["b_skip"], cu["b_out"], A)
    skips = cu["skips"].clone()
    st.layer(packed, cu["b_conv"], bso, d, skips, skips_init=skips_init, write_x=write_x)
    torch.cuda.synchronize()
    return words_in.cpu(), st.x[st.cur].cpu(), st.x[1 - st.cur].cpu(), skips.cpu(), st


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n][6] != "bound"])
def test_exact(dev, name):
    form, (R, G, S, A), B, T, d, dmax, regime, skips_init, write_x = CASES[name]
    dd, emu = case_emulation(name)
    (emu.ex_g if regime == "launch1" else emu.ex).check(name)
    if form == "two":
        g_ws, x_out, skips = run_two(dev, name, dd)
        _assert_equal(g_ws, emu.g, f"{name}: g_ws")
        if regime == "launch1":
            return
        _assert_equal(skips, emu.skips, f"{name}: skips")
        _assert_equal(x_out, emu.x, f"{name}: x'")
        return
    halo = (K - 1) // 2 * dmax
    words_in, words_out, words_other, skips, _ = run_fused(dev, name, dd)
    _assert_equal(words_in, E.pack_words(dd["x"], halo, _tp(T, halo)), f"{name}: packed x")
    _assert_equal(skips, emu.skips, f"{name}: skips")
    if write_x:
        _assert_equal(words_out, E.pack_words(emu.x, halo, _tp(T, halo)), f"{name}: packed x' (halos included)")
    else:
        _assert_equal(words_out, words_in, f"{name}: packed x (write_x off leaves the stream)")
        assert int(words_other.abs().sum()) == 0, f"{name}: write_x off wrote the other buffer"


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n][6] == "bound"])
def test_bound(dev, name):
    """fused layer on general data: every skip and x' element within gate_bound of the fp64 layer"""
    form, (R, G, S, A), B, T, d, dmax, _, _, _ = CASES[name]
    dd = case_data(name)
    b_sk, b_x, ref_sk, ref_x = E.gate_bound(dd, d)
    halo = (K - 1) // 2 * dmax
    _, words_out, _, skips, _ = run_fused(dev, name, dd)
    xo = E.unpack_words(words_out, B, R, halo, _tp(T, halo), T)
    for what, v, ref, bound in (("skips", skips, ref_sk, b_sk), ("x'", xo, ref_x, b_x)):
        r = (v.double() - ref).abs() / bound
        assert float(r.max()) <= 1.0, f"{name}: {what} error {float(r.max()):.3f} x the gate bound at {r.argmax().item()}"


# ---------------------------------------------------------------------------------------------------- gate readout
PROBE_SAT = [0.0, 20.0, -20.0, 64.0, -64.0, 100.0, -100.0, 128.0, -128.0, 1000.0, -1000.0]


def probe_inputs(H, T, gen):
    """(a, b) fp32 (1, H, T) pairs: a sweeps every multiple of 2^-8 in [-50, 50] (b random on that grid), then b does,
    then every pair of saturated values; fits_split holds for all of them."""
    n = H * T
    full = torch.arange(-50 * 256, 50 * 256 + 1, dtype=torch.float64) / 256
    rnd = lambda m: full[torch.randint(0, len(full), (m,), generator=gen)]
    sat = torch.tensor(PROBE_SAT, dtype=torch.float64)
    sa, sb = torch.meshgrid(sat, sat, indexing="ij")
    a = torch.cat([full, rnd(len(full)), sa.reshape(-1)])
    b = torch.cat([rnd(len(full)), full, sb.reshape(-1)])
    assert len(a) <= n
    a = torch.cat([a, rnd(n - len(a))]).float().reshape(1, H, T)
    b = torch.cat([b, rnd(n - len(b))]).float().reshape(1, H, T)
    assert E.fits_split(a) and E.fits_split(b)
    return a, b


EPS_G = 2.0 ** -20  # gate error budget of the readout


def _probe_check(form, a, b, z_read, report):
    """z_read = hi + lo of the device's gate: the identities exactly, every element within EPS_G (plus what the split
    can move) and within the derived gate_fast_bound (fused)."""
    ref = E.gate_fp64(a, b)
    table = E.gate_table(form)
    ta, sg = E.EXACT_TANH[form], E.EXACT_SIGMOID[form]
    cls = torch.isin(a, torch.tensor(list(ta))) & torch.isin(b, torch.tensor(list(sg)))
    if form == "fused":
        cls |= a == 0
    assert int(cls.sum()) > 0
    exact = table(a[cls], b[cls])
    _assert_equal(z_read[cls], exact.float(), f"{form} gate identities")
    err = (z_read.double() - ref).abs()
    allow = E.split_bound(ref, torch.full_like(ref, EPS_G))
    assert float((err / allow).max()) <= 1.0, f"{form} gate: error {float(err.max()):.3e} beyond 2^-20"
    if form == "fused":
        zero = torch.zeros_like(a, dtype=torch.float64)
        eb = E.split_bound(ref, E.gate_fast_bound(a.double(), b.double(), zero, zero))
        assert float((err / eb).max()) <= 1.0, f"fused gate beyond gate_fast_bound: {float((err / eb).max()):.3f}"
    near = (ref - ref.float().to(torch.bfloat16).double()).abs() < 2.0 ** -30  # the split loses nothing there
    report[form] = (float(err.max()), float(err[near].max()) if near.any() else 0.0)


def test_gate_readout(dev):
    """W_conv = 0, W_aux = I, W_skip = I, no bias, zero skips: skips = hi(z) + lo(z) of the device's own gate at
    g = c, through both forms, and tanhf * sigmoidf_ in full fp32 through pwgb_gate_forward."""
    from parallelwavegan_b200 import capi, ops

    R, G, S, A = V1
    H, T = G // 2, 1024
    a, b = probe_inputs(H, T, torch.Generator().manual_seed(11))
    c = torch.cat([a, b], 1)
    base = dict(x=E.grid_values((1, R, T), torch.Generator().manual_seed(12), 1.0, hmax=3), c=c, w_conv=torch.zeros(G, R, K),
                b_conv=None, w_aux=torch.eye(G), w_skip=torch.eye(S, H), w_out=torch.zeros(R, H), b_skip=None, b_out=None,
                skips=torch.zeros(1, S, T))
    report = {}
    CASES["_probe_fused"] = ("fused", V1, 1, T, 1, 1, "probe", True, False)
    CASES["_probe_two"] = ("two", V1, 1, T, 1, None, "probe", False, True)
    try:
        _, _, _, sk_f, _ = run_fused(dev, "_probe_fused", base)
        g_ws, _, sk_t = run_two(dev, "_probe_two", base)
    finally:
        del CASES["_probe_fused"], CASES["_probe_two"]
    _assert_equal(g_ws, c, "probe: g = c")
    _probe_check("fused", a, b, sk_f, report)
    _probe_check("two", a, b, sk_t, report)
    z = torch.empty(1, H, T, device=dev)
    rc = capi.lib().pwgb_gate_forward(_p(c.to(dev)), _p(z), 1, H, T, ops._stream())
    capi.check(rc, "pwgb_gate_forward")
    z = z.cpu()
    ref = E.gate_fp64(a, b)
    for (k, v) in [((20.0, 20.0), 1.0), ((-20.0, 20.0), -1.0), ((20.0, 0.0), 0.5), ((0.0, 0.0), 0.0), ((20.0, -100.0), 0.0)]:
        m = (a == k[0]) & (b == k[1])
        assert int(m.sum()) > 0 and bool((z[m] == v).all()), f"tanhf * sigmoidf_{k} != {v}: {z[m][:4].tolist()}"
    err = float((z.double() - ref).abs().max())
    assert err <= EPS_G, f"tanhf * sigmoidf_: max error {err:.3e} beyond 2^-20"
    print(f"\n[gate] max |readout - fp64|, all / where the split is exact: fused {report['fused'][0]:.3e} / "
          f"{report['fused'][1]:.3e}, two-launch {report['two'][0]:.3e} / {report['two'][1]:.3e}; "
          f"pwgb_gate_forward (full fp32) {err:.3e}")


# ---------------------------------------------------------------------------------------------------- packing helpers
@pytest.mark.parametrize("R,A,T,dmax,B", [(64, 80, 515, 512, 2), (32, 16, 1, 1, 1), (96, 48, 256, 4, 2), (64, 128, 129, 64, 0)])
def test_pack_helpers(dev, R, A, T, dmax, B):
    """pack_x / pack_c / first_conv words equal pack_words (zero halos, zero conditioning tail on [T, Tc), A % 32 = 16
    padded to whole 8-channel groups) and unpack_x(pack_x(x)) == hi + lo"""
    from parallelwavegan_b200 import ops

    G = 128 if R != 32 else 64
    S = G - R
    gen = torch.Generator().manual_seed(R * 1000 + A + T)
    x = torch.randn(B, R, T, generator=gen)
    c = torch.randn(B, A + 8, T, generator=gen)[:, :A] if B else torch.zeros(B, A, T)
    st = ops.WnStack(B, T, R, G, S, A, K, dmax, dev)
    halo = (K - 1) // 2 * dmax
    st.pack_x(x.to(dev))
    st.pack_c(torch.cat([c, torch.randn(B, 8, T, generator=gen)], 1).to(dev))  # extra channels past A are ignored
    _assert_equal(st.x[st.cur].cpu(), E.pack_words(x, halo, _tp(T, halo)), "pack_x")
    _assert_equal(st.c.cpu(), E.pack_words(c, 0, _tp(T, 0)), "pack_c")
    hi, lo = E.split(x)
    _assert_equal(st.unpack_x().cpu(), hi + lo, "unpack_x")
    cin = 4
    zin = E.grid_values((B, cin, T), gen, 1.0, hmax=3, lo=False)  # integer z: the fma chain is exact (16 bits)
    w = E.grid_values((R, cin), gen, 2.0 ** -2, hmax=3)
    bias = E.grid_values((R,), gen, 2.0 ** -1, hmax=3)
    st.first_conv(zin.to(dev), w.to(dev), bias.to(dev))
    ref = (torch.einsum("rc,bct->brt", w.double(), zin.double()) + bias.double().reshape(1, -1, 1)).float()
    _assert_equal(st.x[st.cur].cpu(), E.pack_words(ref, halo, _tp(T, halo)), "first_conv")


# ---------------------------------------------------------------------------------------------------- pwgb_gate_*
GATE_ULP = 16  # tanhf 2 ulp, __expf 2 + 1.173 |v| ulp at |v| <= 8, two roundings


@pytest.mark.parametrize("T,off", [(1024, 0), (1023, 0), (1024, 1), (5, 0)])
def test_gate_forward_backward(dev, T, off):
    """pwgb_gate_forward / pwgb_gate_backward per element against fp64: z within GATE_ULP ulp of |z|; the gradients
    within GATE_ULP ulp of |go| (1 - tanh^2 and 1 - sigmoid cancel near saturation, so the budget is absolute in go).
    T % 4 == 0 with aligned rows takes the float4 path, T % 4 != 0 or a misaligned view the scalar one."""
    from parallelwavegan_b200 import capi, ops

    B, H = 2, 48
    gen = torch.Generator().manual_seed(T + off)
    g = (torch.rand(B, 2 * H, T, generator=gen) * 16 - 8).float()
    g[0, 0, : min(T, 4)] = torch.tensor([0.0, 20.0, -20.0, 8.0])[: min(T, 4)]
    gz = torch.randn(B, H, T, generator=gen)

    def at(t):
        buf = torch.zeros(t.numel() + off, device=dev)
        v = buf[off:].view(t.shape)
        v.copy_(t)
        return v

    gd, gzd = at(g), at(gz)
    z, gg = at(torch.zeros(B, H, T)), at(torch.zeros(B, 2 * H, T))
    L = capi.lib()
    capi.check(L.pwgb_gate_forward(_p(gd), _p(z), B, H, T, ops._stream()), "pwgb_gate_forward")
    capi.check(L.pwgb_gate_backward(_p(gd), _p(gzd), _p(gg), B, H, T, ops._stream()), "pwgb_gate_backward")
    torch.cuda.synchronize()
    a, s = g[:, :H].double(), g[:, H:].double()
    ta, sg = torch.tanh(a), torch.sigmoid(s)
    ulp = GATE_ULP * 2.0 ** -23
    zr = ta * sg
    assert float(((z.cpu().double() - zr).abs() / (ulp * zr.abs() + 2.0 ** -40)).max()) <= 1.0, "gate_forward"
    go = gz.double()
    da, ds = go * sg * (1 - ta * ta), go * ta * sg * (1 - sg)
    ggc = gg.cpu().double()
    for what, v, r in (("d a", ggc[:, :H], da), ("d b", ggc[:, H:], ds)):
        e = (v - r).abs() / (ulp * (r.abs() + go.abs()) + 2.0 ** -40)
        assert float(e.max()) <= 1.0, f"gate_backward {what}: {float(e.max()):.3f} x the budget"
