"""The exact fp64 reference of the FFMA kernels (oracle/ffma_exact.py) checked on the CPU, and the tables of
tests/test_gpu_ffma_exact.py.

- the reference is right: against F.conv2d / F.conv_transpose1d / conv_transpose2d / torch.nn.grad.conv1d_weight /
  fp64 autograd, and every adjoint satisfies <A x, y> == <x, A^T y> exactly on grid data;
- the premise holds: on guarded data fp32 sums of the terms in shuffled orders equal the reference, and lo parts on
  both operands fail the guard;
- the data have teeth: for every table row, plausible kernel mistakes applied to the reference change the result;
- check_coverage() of the GPU tables."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import bf16x3 as E
from oracle import ffma_exact as X


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _dot(a, b):
    return float((a.double() * b.double()).sum())


# ---------------------------------------------------------------------------------------------------- the reference is right
@pytest.mark.parametrize("P,S,L", [(2, 3, 301), (3, 3, 299), (5, 3, 300), (1, 2, 200)])
def test_period_conv_is_conv2d(P, S, L):
    """the period-view conv (with the t_valid reflect extension) is a (K, 1) Conv2d over the reflect-padded signal"""
    g = _gen(P * 100 + L)
    x = E.grid_values((2, 4, L), g, 1.0, 3)
    w = E.grid_values((6, 2, 5), g, 2.0 ** -4, 3, lo=False)
    y, ex = X.conv1d(x, w, stride=S, padding=2, groups=2, period=P, pre_slope=0.5)
    assert ex.ok
    rows = -(-L // P)
    xe = F.pad(E.lrelu(x, 0.5).double(), (0, rows * P - L), mode="reflect")
    ref = F.conv2d(xe.view(2, 4, rows, P), w.double().unsqueeze(-1), stride=(S, 1), padding=(2, 0), groups=2)
    assert torch.equal(y.double(), ref if P > 1 else ref[..., 0])


def test_t_valid_extension_is_reflect_pad():
    x = torch.arange(10.0).view(1, 1, 10)
    c = X.columns(x, 4)  # rows 3: 10 -> 12 samples, x_ext[10 + m] = x[8 - m]
    assert torch.equal(c.permute(1, 2, 0).reshape(-1), torch.tensor([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 8, 7.0]))


@pytest.mark.parametrize("mode,pad", [("reflect", (3, 5)), ("replicate", (4, 1)), ("zero", (0, 6))])
def test_conv_padding_modes(mode, pad):
    g = _gen(3)
    x = E.grid_values((2, 3, 40), g, 1.0, 3)
    w = E.grid_values((4, 3, 7), g, 2.0 ** -4, 3, lo=False)
    y, _ = X.conv1d(x, w, padding=pad, dilation=2, pad_mode=mode)
    xp = F.pad(x.double(), pad) if mode == "zero" else F.pad(x.double(), pad, mode=mode)
    assert torch.equal(y.double(), F.conv1d(xp, w.double(), dilation=2))


@pytest.mark.parametrize("G,P,s,K,p,op", [(4, 1, 4, 8, 2, 0), (1, 3, 3, 5, 2, 1), (1, 1, 2, 4, 1, 1), (16, 1, 2, 41, 20, 1)])
def test_conv_transpose_is_the_pytorch_conv_transpose(G, P, s, K, p, op):
    """the virtual conv + pixel shuffle of the FFMA kernel equals F.conv_transpose1d / conv_transpose2d"""
    g = _gen(G * 10 + P)
    cin = 2 * G * 2 if G > 1 else 6
    x = E.grid_values((2, cin, 30) + ((P,) if P > 1 else ()), g, 1.0, 3)
    w = E.grid_values((cin, 8 // min(G, 8) if G > 1 else 5, K), g, 2.0 ** -4, 3, lo=False)
    b = E.grid_values((w.shape[1] * G,), g, 2.0 ** -4, 3)
    y, ex = X.conv_transpose1d(x, w, b, stride=s, padding=p, output_padding=op, groups=G, period=P, pre_slope=0.5)
    assert ex.ok
    xa = E.lrelu(x, 0.5).double()
    if P > 1:
        ref = F.conv_transpose2d(xa, w.double().unsqueeze(-1), b.double(), stride=(s, 1), padding=(p, 0), output_padding=(op, 0))
    else:
        ref = F.conv_transpose1d(xa, w.double(), b.double(), stride=s, padding=p, output_padding=op, groups=G)
    assert torch.equal(y.double(), ref)


@pytest.mark.parametrize("S,D,G,P,pl", [(1, 2, 1, 1, 2), (2, 1, 4, 1, 2), (3, 1, 1, 3, 2), (3, 1, 1, 5, 2)])
def test_wgrad_is_the_weight_gradient(S, D, G, P, pl):
    g = _gen(S * 7 + P)
    B, cin, cout, K, L = 2, 8, 8, 5, 301
    x = E.grid_values((B, cin, L), g, 1.0, 2)
    xa = E.lrelu(x, 0.5).double()
    rows = -(-L // P)
    xe = F.pad(xa, (0, rows * P - L), mode="reflect")
    t_out = (rows + 2 * pl - D * (K - 1) - 1) // S + 1
    gy = E.grid_values((B, cout, t_out) + ((P,) if P > 1 else ()), g, 2.0 ** -4, 2, lo=False)
    dw, ex = X.conv1d_wgrad(x, gy, K, stride=S, pad_left=pl, dilation=D, groups=G, period=P, x_slope=0.5, g_slope=0.25)
    assert ex.ok
    ga = E.lrelu(gy, 0.25).double()
    wr = torch.zeros(cout, cin // G, K, dtype=torch.float64, requires_grad=True)
    if P > 1:
        F.conv2d(xe.view(B, cin, rows, P), wr.unsqueeze(-1), stride=(S, 1), padding=(pl, 0), groups=G).backward(ga)
    else:
        F.conv1d(xe, wr, stride=S, padding=pl, dilation=D, groups=G).backward(ga)
        assert torch.equal(dw.double(), torch.nn.grad.conv1d_weight(xe, wr.shape, ga, stride=S, padding=pl, dilation=D, groups=G))
    assert torch.equal(dw.double(), wr.grad)


def test_adjoints_are_exact_on_grid_data():
    g = _gen(11)
    # conv <-> conv-transpose (stride, groups, padding) and conv <-> weight gradient
    x = E.grid_values((2, 8, 61), g, 1.0, 3)
    w = E.grid_values((12, 2, 7), g, 2.0 ** -4, 3, lo=False)
    y, _ = X.conv1d(x, w, stride=3, padding=3, groups=4)
    gy = E.grid_values(tuple(y.shape), g, 1.0, 3, lo=False)
    op = 61 - ((y.shape[-1] - 1) * 3 - 6 + 7)
    gx, _ = X.conv_transpose1d(gy, w, stride=3, padding=3, output_padding=op, groups=4)
    assert _dot(y, gy) == _dot(x, gx)
    dw, _ = X.conv1d_wgrad(x, gy, 7, stride=3, pad_left=3, groups=4)
    assert _dot(y, gy) == _dot(w, dw)
    # upsample FIR: forward, x adjoint, filter adjoint
    f = E.grid_values((9,), g, 2.0 ** -3, 3, lo=False)
    xu = E.grid_values((2, 3, 20), g, 1.0, 3)
    yu, _ = X.upsample_fir(xu, f, 4)
    gu = E.grid_values(tuple(yu.shape), g, 1.0, 3, lo=False)
    assert _dot(yu, gu) == _dot(xu, X.upsample_fir_backward_x(gu, f, 4)[0]) == _dot(f, X.upsample_fir_backward_f(xu, gu, 4)[0])
    # gathers
    xs = E.grid_values((2, 8, 30, 3), g, 1.0, 3)
    ys, _ = X.s2d(xs, 2, 3, 2, 11, 3, 16)
    gs = E.grid_values(tuple(ys.shape), g, 1.0, 3)
    gs.view(2, 2, 16, 11, 3)[:, :, 12:] = 0  # the zero channels have no adjoint
    assert _dot(ys, gs) == _dot(xs, X.s2d_backward(gs, tuple(xs.shape), 2, 3, 2, 3, 16)[0])
    for mode in ("reflect", "replicate"):
        xp = E.grid_values((2, 3, 9), g, 1.0, 3)
        yp, _ = X.pad1d(xp, 8, 3, mode)
        gp = E.grid_values(tuple(yp.shape), g, 1.0, 3)
        assert _dot(yp, gp) == _dot(xp, X.pad1d_backward(gp, 9, 8, 3, mode)[0])
    for k, s, p, inc in ((4, 2, 2, True), (4, 2, 1, False)):
        xa = E.grid_values((2, 3, 101), g, 1.0, 3)
        t_out = (101 + 2 * p - k) // s + 1
        ga = 12.0 * E.grid_values((2, 3, t_out), g, 1.0, 3)
        div = X._pool_div(101, t_out, k, s, p, inc).double()
        A = X._pool_matrix(101, k, s, p)
        lhs = float((torch.einsum("bci,oi->bco", xa.double(), A) * ga.double() / div).sum())
        assert lhs == _dot(xa, X.avg_pool1d_backward(ga, 101, k, s, p, inc)[0])


# ---------------------------------------------------------------------------------------------------- the premise holds
def _terms(x, w, K):
    """every product of a valid stride-1 conv as (B, cout, t_out, cin * K) fp64 (exact: products of two fp32 values)"""
    u = x.double().unfold(2, K, 1)
    return torch.einsum("bctk,ock->botck", u, w.double()).reshape(x.shape[0], w.shape[0], u.shape[2], -1)


def test_fp32_sums_in_any_order_equal_the_reference_on_guarded_data():
    g = _gen(5)
    x = E.grid_values((1, 64, 40), g, 1.0, hmax=3)
    w = E.grid_values((16, 64, 11), g, 2.0 ** -4, hmax=3, lo=False)
    y, ex = X.conv1d(x, w)
    assert ex.ok and ex.bits > 16
    terms = _terms(x, w, 11)
    assert torch.equal(terms.float().double(), terms)  # every product is exact in fp32
    terms = terms.float()
    for seed in range(3):
        perm = torch.randperm(terms.shape[-1], generator=_gen(seed))
        acc = torch.zeros(terms.shape[:-1])
        for blk in terms[..., perm].split(8, dim=-1):  # fp32 partial sums of 8 products, then a running sum
            acc = acc + blk.sum(-1)
        assert torch.equal(acc, y)


def test_guard_rejects_lo_parts_on_both_operands():
    g = _gen(6)
    x = E.grid_values((1, 64, 40), g, 1.0, hmax=3)
    w_lo = E.grid_values((16, 64, 11), g, 2.0 ** -4, hmax=3)
    _, ex = X.conv1d(x, w_lo)
    assert not ex.ok
    # and the products are not all exact in fp32 any more (24-bit products of two 12-bit values are; sums are not)
    terms = _terms(x, w_lo, 11)
    exact = terms.sum(-1)
    seq = torch.zeros(terms.shape[:-1])
    for i in range(terms.shape[-1]):
        seq = seq + terms[..., i].float()
    assert not torch.equal(seq.double(), exact)


# ---------------------------------------------------------------------------------------------------- the data have teeth
def _hi(t):
    """the operand with its lo part dropped"""
    return E.split(t)[0]


def _changes(ref, mutated, what):
    assert not torch.equal(ref, mutated[0] if isinstance(mutated, tuple) else mutated), what


def _conv_mutations(T, name):
    r = T.CONV[name]
    d, ref, _ = T.conv_case(name)
    p, G = r["plan"], r["G"]
    out = {"last tap dropped": T.conv_ref(r, dict(d, w=F.pad(d["w"][..., :-1], (0, 1))))}
    pl, pr = r["pad"]
    out["left padding off by one"] = T.conv_ref(r, d, pad=(pl + 1, pr - 1) if pr > 0 else (pl - 1, pr + 1))
    if r["mode"] != "zero":
        out["reflect / replicate swapped"] = T.conv_ref(r, d, mode={"reflect": "replicate", "replicate": "reflect"}[r["mode"]])
    cin_g = r["cin"] // G
    if p["kernel"] == 0 and cin_g > 1:
        ci_t = p.get("CI_T", min(16, cin_g))
        c0 = (cin_g - 1) // ci_t * ci_t if cin_g > ci_t else cin_g - 1
        x = d["x"].clone().view(r["B"], G, cin_g, -1)
        x[:, :, c0:] = 0
        out["last input-channel chunk dropped"] = T.conv_ref(r, dict(d, x=x.view_as(d["x"])))
    if G > 1:
        out["group offset wrong"] = T.conv_ref(r, dict(d, w=d["w"].roll(r["cout"] // G, 0)))
    k = "x" if r["lo"] == "x" else "w"
    out["lo part dropped"] = T.conv_ref(r, dict(d, **{k: _hi(d[k])}))
    return ref, out


def _wgrad_mutations(T, name):
    r = T.WGRAD[name]
    d, ref, _ = T.wgrad_case(name)
    out = {"last tap dropped": (torch.cat([ref[..., :-1], torch.zeros_like(ref[..., -1:])], -1),)}
    out["left padding off by one"] = T.wgrad_ref(r, d, pl=r["pl"] + 1)
    if r["mode"] != "zero":
        out["reflect / replicate swapped"] = T.wgrad_ref(r, d, mode={"reflect": "replicate", "replicate": "reflect"}[r["mode"]])
    chunk = 1024 if r["plan"]["path"] == 1 else 128
    gy = d["gy"].clone()
    flat = gy.view(r["B"], r["cout"], -1)
    n = flat.shape[-1]
    flat[..., (n - 1) // chunk * chunk:] = 0
    out["last partial time chunk dropped"] = T.wgrad_ref(r, dict(d, gy=gy))
    cin_g, G = r["cin"] // r["G"], r["G"]
    if r["plan"]["path"] == 0 and cin_g > 8:
        x = d["x"].clone().view(r["B"], G, cin_g, -1)
        x[:, :, (cin_g - 1) // 8 * 8:] = 0
        out["last input-channel chunk dropped"] = T.wgrad_ref(r, dict(d, x=x.view_as(d["x"])))
    if G > 1:
        out["group offset wrong"] = T.wgrad_ref(r, dict(d, x=d["x"].roll(cin_g, 1)))
    k = "x" if r["lo"] == "x" else "gy"
    out["lo part dropped"] = T.wgrad_ref(r, dict(d, **{k: _hi(d[k])}))
    return ref, out


def _rows():
    import test_gpu_ffma_exact as T

    return T


def _all_rows():
    T = _rows()
    return ([("conv", n) for n in T.CONV] + [("wgrad", n) for n in T.WGRAD] + [("convtr", n) for n in T.CONVTR]
            + [("fir", n) for n in T.FIR] + [("bias", n) for n in T.BIAS] + [("gather", n) for n in T.GATHER]
            + [("act", n) for n in T.ACT])


@pytest.mark.parametrize("family,name", _all_rows())
def test_mutations_change_the_reference(family, name):
    """plausible kernel mistakes, applied to the reference, change at least one element of every table row"""
    T = _rows()
    if family == "conv":
        ref, out = _conv_mutations(T, name)
    elif family == "wgrad":
        ref, out = _wgrad_mutations(T, name)
    elif family == "convtr":
        row = T.CONVTR[name]
        d, ref, _ = T._draw(name, lambda g, h, z: (lambda d_: (d_,) + T.convtr_ref(row, d_))(T.convtr_inputs(row, g, h, z)),
                            row[1] // row[7] * math.ceil(row[3] / row[4]))
        k = "x" if row[10] == "x" else "w"
        out = {"last tap dropped": T.convtr_ref(row, dict(d, w=F.pad(d["w"][..., :-1], (0, 1)))),
               "lo part dropped": T.convtr_ref(row, dict(d, **{k: _hi(d[k])}))}
        if row[7] > 1:
            out["group offset wrong"] = T.convtr_ref(row, dict(d, w=d["w"].roll(row[1] // row[7], 0)))
    elif family == "fir":
        row = T.FIR[name]
        d, ref, _ = T.fir_case(name)
        op, lo = row[0], row[6]
        k = {("fwd", "x"): "x", ("fwd", "f"): "f", ("dx", "x"): "gy", ("dx", "f"): "f", ("df", "x"): "x", ("df", "f"): "gy"}[(op, lo)]
        out = {"lo part dropped": T.fir_ref(row, dict(d, **{k: _hi(d[k])}))}
        if op != "df":
            out["last tap dropped"] = T.fir_ref(row, dict(d, f=F.pad(d["f"][:-1], (0, 1))))
        else:
            gy = d["gy"].clone()
            gy[-1, row[2] - 1] = 0  # the last row (the last cluster rank's share) dropped
            out["last row dropped"] = T.fir_ref(row, dict(d, gy=gy))
    elif family == "bias":
        row = T.BIAS[name]
        d = T.bias_inputs(row, _gen(len(name) * 7919))
        ref, _ = X.bias_grad(d["g"], d["prev"])
        g = d["g"].clone()
        g[..., -(g.shape[-1] % 4 or 4):] = 0  # the scalar tail / the last float4 of every row dropped
        out = {"last partial chunk dropped": X.bias_grad(g, d["prev"])}
        if row[5]:
            out["lo part dropped"] = X.bias_grad(_hi(d["g"]), d["prev"])
    elif family == "gather":
        row = T.GATHER[name]
        d = T.gather_inputs(row, _gen(len(name)))
        ref, _ = T.gather_ref(row, d, False)
        if row[0] == "s2d":
            out = {"left padding off by one": T.gather_ref(row[:7] + (row[7] + 1,) + row[8:], d, False)}
            if row[3] > 1:
                out["group offset wrong"] = T.gather_ref(row, dict(d, x=d["x"].roll(row[2] // row[3], 1)), False)
        elif row[0] == "pad":
            other = {"reflect": "replicate", "replicate": "reflect"}[row[6]]
            out = {"reflect / replicate swapped": T.gather_ref(row[:6] + (other,), d, False)}
        else:
            out = {"count_include_pad swapped": T.gather_ref(row[:7] + (not row[7],), d, False)}
        out["lo part dropped"] = T.gather_ref(row, dict(d, x=_hi(d["x"])), False)
    else:
        row = T.ACT[name]
        d = T.act_inputs(row, _gen(len(name)))
        ref, _ = X.act_backward(row[0], d["g"], d["ref"], 0.125, 0.5, d["prev"])
        k = "g" if row[1] == "g" else "ref"
        out = {"lo part dropped": X.act_backward(row[0], **dict(dict(g=d["g"], ref=d["ref"]), **{k: _hi(d[k])}), slope=0.125, scale=0.5,
                                                 prev=d["prev"])}
    for what, mutated in out.items():
        _changes(ref, mutated, f"{name}: {what}")


def test_gpu_case_table_covers_every_branch():
    _rows().check_coverage()
