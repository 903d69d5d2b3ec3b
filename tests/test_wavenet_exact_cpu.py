"""The WaveNet layer emulation of oracle/bf16x3.py checked on the CPU, and the case table of
tests/test_gpu_wavenet_exact.py.

- with the lo*lo terms restored, the emulation is the fp64 layer (oracle/ref_ops.wavenet_residual_block);
- on guarded data, fp32 sums of the terms of g in any order equal the emulation (the premise of the exact GPU cases);
- pack_words round-trips and leaves halos, tails and padding channels zero;
- the data builders produce g == 0, or gate inputs in the exact classes;
- the gate bound is not vacuous: on the bound-regime data every modelled kernel mutation exceeds it by 4x somewhere,
  while an fp32-exact gate stays within it;
- the GPU case table covers every class it is meant to."""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from oracle import bf16x3 as E
from oracle import ref_ops
import test_gpu_wavenet_exact as W


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _weights(d):
    G = d["w_conv"].shape[0]
    w = {"b.conv.weight": d["w_conv"].double(), "b.conv1x1_aux.weight": d["w_aux"].double().reshape(G, -1, 1),
         "b.conv1x1_skip.weight": d["w_skip"].double().reshape(d["w_skip"].shape[0], -1, 1),
         "b.conv1x1_out.weight": d["w_out"].double().reshape(d["w_out"].shape[0], -1, 1)}
    if d["b_conv"] is not None:
        w["b.conv.bias"] = d["b_conv"].double()
    if d["b_skip"] is not None:
        w["b.conv1x1_skip.bias"] = d["b_skip"].double()
        w["b.conv1x1_out.bias"] = d["b_out"].double()
    return w


@pytest.mark.parametrize("form", ["two", "fused"])
def test_emulation_plus_lolo_is_the_fp64_layer(form):
    """saturated data of the fused classes (tanh(-64) = -1, sigmoid(128) = 1 and sigmoid(0) = 0.5 hold in fp64 too, so
    z is exact) with general grid x, W_skip / W_out and biases: skips and x' equal the fp64 layer (x' up to the fp32
    sqrt(1/2), applied to both), and on general grid data g (conv + aux + bias) equals the fp64 conv"""
    B, R, G, S, T, d = 2, 64, 128, 64, 50, 4
    dd = E.saturated_data(_gen(1), B, R, G, S, T, "fused")
    emu = E.wavenet_layer(dd["x"], dd["c"], dd["w_conv"], dd["b_conv"], dd["w_aux"], dd["w_skip"], dd["b_skip"], dd["w_out"],
                          dd["b_out"], dilation=d, form=form, gate=E.gate_fp64, lolo=True)
    emu.ex.check()
    xr, sr = ref_ops.wavenet_residual_block(_weights(dd), "b", dd["x"].double(), dd["c"].double(), d, 3)
    assert torch.equal(emu.skips, sr.float())
    assert torch.equal(emu.x, (xr / math.sqrt(0.5) * E.SQRT_HALF).float())
    # general grid data: g (conv + aux + bias) is the fp64 conv exactly
    gen = _gen(3)
    x, c = E.grid_values((B, R, T), gen, 1.0, hmax=3), E.grid_values((B, 80, T), gen, 1.0, hmax=3)
    wc, wa = E.grid_values((G, R, 3), gen, 2.0 ** -3, hmax=3), E.grid_values((G, 80), gen, 2.0 ** -3, hmax=3)
    bc = E.grid_values((G,), gen, 0.5, hmax=3)
    emu = E.wavenet_layer(x, c, wc, bc, wa, dd["w_skip"], None, dd["w_out"], None, dilation=d, form="two", lolo=True)
    emu.ex_g.check()
    ref = F.conv1d(x.double(), wc.double(), bc.double(), padding=d, dilation=d) + F.conv1d(c.double(), wa.double()[..., None])
    assert torch.equal(emu.g, ref.float())  # both the exact fp64 value, rounded once


def test_shuffled_fp32_sums_equal_the_emulation():
    """every term of g (three bf16 products per conv tap and aux channel, and the bias) summed in fp32 in a random
    order per element equals the emulated g on guarded data"""
    B, R, G, A, T, d = 2, 32, 64, 32, 40, 3
    gen = _gen(4)
    x, c = E.grid_values((B, R, T), gen, 1.0, hmax=2), E.grid_values((B, A, T), gen, 1.0, hmax=2)
    wc, wa = E.grid_values((G, R, 3), gen, 2.0 ** -3, hmax=2), E.grid_values((G, A), gen, 2.0 ** -3, hmax=2)
    bc = E.grid_values((G,), gen, 0.5, hmax=3)
    emu = E.wavenet_layer(x, c, wc, bc, wa, torch.zeros(16, G // 2), None, torch.zeros(R, G // 2), None, dilation=d, form="two")
    emu.ex_g.check()
    xh, xl = E.split(x)
    ch, cl = E.split(c)
    wh, wl = E.split(wc)
    ah, al = E.split(wa)
    xs = [F.pad(t, (d, d)).unfold(2, 2 * d + 1, 1)[..., ::d] for t in (xh, xl)]  # (B, R, T, 3)
    terms = []
    for xa, wb in ((xs[0], wh), (xs[1], wh), (xs[0], wl)):
        terms.append((xa.unsqueeze(1) * wb.reshape(1, G, R, 1, 3)).permute(0, 1, 3, 2, 4).reshape(B, G, T, -1))
    for ca, wb in ((ch, ah), (cl, ah), (ch, al)):
        terms.append((ca.unsqueeze(1) * wb.reshape(1, G, A, 1)).permute(0, 1, 3, 2))
    terms.append(bc.reshape(1, G, 1, 1).expand(B, G, T, 1))
    terms = torch.cat(terms, -1).float()
    perm = torch.argsort(torch.rand(terms.shape, generator=gen), -1)
    terms = torch.gather(terms, -1, perm)
    acc = torch.zeros(B, G, T, dtype=torch.float32)
    for i in range(terms.shape[-1]):
        acc = acc + terms[..., i]
    assert torch.equal(acc, emu.g)


@pytest.mark.parametrize("B,C,T,halo,t_pad", [(2, 64, 300, 16, 544), (1, 80, 5, 0, 256), (0, 64, 10, 2, 260)])
def test_pack_words_round_trip(B, C, T, halo, t_pad):
    x = torch.randn(B, C, T, generator=_gen(5))
    w = E.pack_words(x, halo, t_pad)
    ng = (C + 7) // 8
    assert w.dtype == torch.int32 and w.numel() == B * 2 * ng * t_pad * 4
    hi, lo = E.split(x)
    assert torch.equal(E.unpack_words(w, B, C, halo, t_pad, T), hi + lo)
    img = w.view(torch.int16).reshape(B, 2, ng, t_pad, 8)
    assert int(img[:, :, :, :halo].abs().sum()) == 0 and int(img[:, :, :, halo + T:].abs().sum()) == 0
    if C % 8:
        assert int(img[:, :, -1, :, C % 8:].abs().sum()) == 0
    # channel 2i sits in the low half of word i
    if B:
        assert int(w[0] & 0xFFFF) == int(hi[0, 0, 0].to(torch.bfloat16).view(torch.int16)) & 0xFFFF or halo > 0


@pytest.mark.parametrize("lo_on", ["x", "w"])
def test_zero_target_builder(lo_on):
    for R, G, d in ((64, 128, 1), (96, 128, 512), (32, 64, 8)):
        dd = E.zero_target_data(_gen(6), 2, R, G, G - R if G - R else 32, 300, 3, d, lo_on=lo_on)
        emu = E.wavenet_layer(dd["x"], dd["c"], dd["w_conv"], dd["b_conv"], dd["w_aux"], dd["w_skip"], dd["b_skip"],
                              dd["w_out"], dd["b_out"], dilation=d, form="fused", gate=E.gate_table("fused"))
        assert E.fits_split(dd["c"]) and bool((emu.g == 0).all())
        assert bool((emu.z == 0).all())
        emu.ex.check()
        other = "w" if lo_on == "x" else "x"
        src = dd["x"] if other == "x" else dd["w_conv"]
        assert bool((E.split(src)[1] == 0).all()) and bool((E.split(dd["x"] if lo_on == "x" else dd["w_conv"])[1] != 0).any())


@pytest.mark.parametrize("form", ["two", "fused"])
def test_saturated_builder(form):
    dd = E.saturated_data(_gen(7), 2, 64, 128, 64, 400, form)
    H = 64
    a, b = dd["c"][:, :H], dd["c"][:, H:]
    assert set(a.unique().tolist()) == set(E.EXACT_TANH[form]) and set(b.unique().tolist()) == set(E.EXACT_SIGMOID[form])
    z = E.gate_table(form)(a, b)
    want = {0.0, -0.5, -1.0} if form == "fused" else {0.0, 0.5, -0.5, 1.0, -1.0}
    assert set(z.unique().tolist()) == want
    # the table agrees with the fp64 gate wherever the fp64 gate is exact in fp32 (sigmoid(-100) is not: the device's
    # __expf overflows to inf there and returns 0)
    ok = b != -100
    ref = E.gate_fp64(a, b).float().double()
    if form == "two":
        assert torch.equal(z[ok], ref[ok])


C1 = 2 / math.log(2)


def _clamp20(a, b):
    e = torch.exp2(torch.clamp(C1 * a, max=20.0))
    return (e - 1) / (e + 1) * torch.sigmoid(b)


MUTATIONS = {
    "drop x_lo w_hi conv product": dict(drop=("x_lo_w_hi",)),
    "drop x_lo in the x' epilogue": dict(drop=("x_lo",)),
    "drop z_lo w_hi skip / out product": dict(drop=("z_lo_w_hi",)),
    "gate_fast clamp 43.28 -> 20": dict(gate=_clamp20),
}


@pytest.mark.parametrize("name", [n for n in W.CASES if W.CASES[n][6] == "bound"])
def test_gate_bound_is_not_vacuous(name):
    form, shape, B, T, d, _, _, _, _ = W.CASES[name]
    dd = W.case_data(name)
    b_sk, b_x, ref_sk, ref_x = E.gate_bound(dd, d)
    args = [dd[k] for k in ("x", "c", "w_conv", "b_conv", "w_aux", "w_skip", "b_skip", "w_out", "b_out")]

    def ratio(kw):
        emu = E.wavenet_layer(*args, dilation=d, form="fused", skips=dd["skips"], **kw)
        return max(float(((emu.skips.double() - ref_sk).abs() / b_sk).max()), float(((emu.xw.double() - ref_x).abs() / b_x).max()))

    assert ratio({}) <= 1.0  # an ideal device: the fp64 gate rounded to fp32
    for what, kw in MUTATIONS.items():
        assert ratio(kw) >= 4.0, f"{name}: {what} exceeds the bound by only {ratio(kw):.2f}x"


def test_gate_bound_holds_on_the_gate_fast_model():
    """the bound holds for an fp64 model of gate_fast with its fp32 constants, clamp and every rounding"""
    gen = _gen(8)
    g = (torch.randint(-50 * 256, 50 * 256 + 1, (2, 200000), generator=gen).double() / 256).float()
    bias = E.grid_values((2, 200000), gen, 2.0 ** -1, hmax=3)
    ga, gb = g.double()
    ba, bb = bias.double()
    f = lambda v: torch.tensor(v, dtype=torch.float32).double() if not torch.is_tensor(v) else v.float().double()
    pa = torch.minimum(f(ga * E.LOG2E2 + f(ba * E.LOG2E2)), torch.tensor(E.CLAMP_A, dtype=torch.float64))
    pb = f(gb * E.NLOG2E + f(bb * E.NLOG2E))
    ea, eb = f(torch.exp2(pa)), f(torch.exp2(pb))
    z = f(f(ea - 1) / f(f(ea + 1) * f(1 + eb)))
    ref = E.gate_fp64(ga + ba, gb + bb)
    bound = E.gate_fast_bound(ga, gb, ba, bb)
    assert float(((z - ref).abs() / bound).max()) <= 1.0


def test_case_table_covers_every_class():
    cases = W.CASES.values()
    exact = [c for c in cases if c[6] in ("zero_x", "zero_w", "sat")]
    for form in ("two", "fused"):
        for regime in ("zero_x", "zero_w", "sat"):
            assert {c[1] for c in exact if c[0] == form and c[6] == regime} & set(W.SHAPES), (form, regime)
        assert set(W.SHAPES) <= {c[1] for c in exact if c[0] == form}, form
        assert any(c[2] == 0 for c in cases if c[0] == form), f"{form}: B = 0"
        assert any(c[2] == 3 and c[3] == 128 * 150 for c in cases if c[0] == form), f"{form}: 150 tiles per sequence"
    fz = [c for c in cases if c[0] == "fused" and c[6] in ("zero_x", "zero_w")]
    assert {1, 2, 8, 64, 128, 256, 512} <= {c[4] for c in fz}
    assert any(c[5] == c[4] for c in fz) and any(c[5] > c[4] for c in fz), "halo tight and loose"
    assert {1, 4, 127, 128, 129, 255, 256, 257, 515} <= {c[3] for c in cases if c[0] == "fused"}
    assert any(c[3] == 100 and c[4] == 512 for c in fz)
    fs = [c for c in cases if c[0] == "fused" and c[6] == "sat"]
    assert {True, False} == {c[7] for c in fs} and False in {c[8] for c in fs}
    assert {1, 2, 8, 64, 128, 256, 512} <= {c[4] for c in cases if c[6] == "launch1"}
    assert {32, 64, 96, 128} <= {c[1][3] for c in cases if c[6] == "launch1"}
    bound = [c for c in cases if c[6] == "bound"]
    assert set(W.SHAPES) <= {c[1] for c in bound} | {W.V1} and any(c[1][3] == 80 for c in bound)
