"""The references and bounds of oracle/glue_exact.py checked on the CPU, over the tables tests/test_gpu_glue_exact.py runs.

- the references are right: against torch's float64 ops, torch.optim.Adam in float64 and oracle/ref_optim.py;
- the bounds are honest: a plain fp32 evaluation of each formula (numpy float32, its own summation order) stays inside
  them, so a correct kernel can;
- the bounds have teeth: each plausible kernel mistake, applied to the reference, moves it by more than the bound at
  some case of the table, so the GPU comparison would have failed;
- the exact data are exact: the preconditions hold on the data the GPU tests use and fail on data that would not be."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import glue_exact as G
from oracle import ref_optim

f32 = np.float32


def _t(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float64))


def _exceeds(mut, ref, bound):
    """the mutated reference lies outside the bound around the true one somewhere"""
    return G.ratio(mut, ref, bound) > 1.0


# ---------------------------------------------------------------------------------------------------- optimizer
@pytest.mark.parametrize("kind,lr,betas,eps,wd", [("adam", 2e-4, (0.5, 0.9), 1e-8, 0.0), ("adam", 2e-4, (0.5, 0.9), 1e-8, 0.01),
                                                  ("radam", 1e-4, (0.9, 0.999), 1e-6, 0.0), ("radam", 1e-2, (0.9, 0.999), 1e-6, 0.01)])
def test_optim_reference_matches_torch_and_ref_optim(kind, lr, betas, eps, wd):
    sizes = [5, 300]
    ps = [t.astype(np.float64) for t in G.optim_random_tensors(sizes, 1, 0)]
    ms = [np.zeros(n) for n in sizes]
    vs = [np.zeros(n) for n in sizes]
    rp = [_t(p).clone() for p in ps]
    rm = [torch.zeros(n, dtype=torch.float64) for n in sizes]
    rv = [torch.zeros(n, dtype=torch.float64) for n in sizes]
    tp = [torch.nn.Parameter(_t(p).clone()) for p in ps]
    topt = torch.optim.Adam(tp, lr=lr, betas=betas, eps=eps, weight_decay=wd) if kind == "adam" else None
    modes = set()
    for t in range(1, 9):
        gs = G.optim_random_tensors(sizes, 2, t)
        for i in range(len(sizes)):
            # the reference rounds its scalars to fp32 like the kernel's arguments: compare at the level of that rounding
            o = G.optim_step(kind, ps[i], gs[i], ms[i], vs[i], t, lr, betas, eps, wd)
            ps[i], ms[i], vs[i] = o["p"], o["m"], o["v"]
            modes.add(o["mode"])
            (ref_optim.adam_step if kind == "adam" else ref_optim.radam_step)(rp[i], _t(gs[i]), rm[i], rv[i], t, lr, betas, eps, wd)
            if topt is not None:
                tp[i].grad = _t(gs[i]).clone()
        if topt is not None:
            topt.step()
        for i in range(len(sizes)):
            np.testing.assert_allclose(ps[i], rp[i].numpy(), rtol=0, atol=2e-6 * t * lr / 1e-4 + 1e-7)
            # 1 - beta formed in fp32 from fp32(beta), as the kernel does: 1 - fp32(0.999) is 1.3e-5 below 0.001
            np.testing.assert_allclose(ms[i], rm[i].numpy(), rtol=3e-5, atol=1e-7)
            np.testing.assert_allclose(vs[i], rv[i].numpy(), rtol=3e-5, atol=1e-9)
            if topt is not None:
                np.testing.assert_allclose(rp[i].numpy(), tp[i].detach().numpy(), rtol=0, atol=1e-12)
    assert modes == ({0} if kind == "adam" else {1, 2})  # RAdam's rectification switches on at step 6


def _optim_f32(kind, p, g, m, v, t, lr, betas, eps, wd, coef):
    """the update in plain fp32, no contraction"""
    p, g, m, v = (np.asarray(a, f32) for a in (p, g, m, v))
    b1, b2, lr_, eps_, wd_ = f32(betas[0]), f32(betas[1]), f32(lr), f32(eps), f32(wd)
    if coef is not None:
        g = g * f32(coef)
    if kind == "adam":
        mode, c1, c2 = 0, f32(lr / (1.0 - betas[0] ** t)), f32(1.0 / np.sqrt(1.0 - betas[1] ** t))
        if wd:
            g = (wd_.astype(np.float64) * p + g).astype(f32)  # fmaf
    else:
        mode, ss = G.radam_mode(t, betas)
        c1, c2 = f32(ss * lr), f32(1)
    m = b1 * m + (f32(1) - b1) * g
    v = b2 * v + (f32(1) - b2) * g * g
    if mode == 0:
        p = p - c1 * (m / (np.sqrt(v) * c2 + eps_))
    else:
        if wd:
            p = p - wd_ * lr_ * p
        p = p - (c1 * (m / (np.sqrt(v) + eps_)) if mode == 1 else c1 * m)
    return p, m, v


@pytest.mark.parametrize("kind,lr,betas,eps,wd,clip", [
    ("adam", 2e-4, (0.5, 0.9), 1e-8, 0.0, None), ("adam", 2e-4, (0.5, 0.9), 1e-8, 0.01, 3.0),
    ("radam", 1e-4, (0.9, 0.999), 1e-6, 0.0, 10.0), ("radam", 1e-4, (0.9, 0.999), 1e-6, 0.01, None)])
def test_optim_bound_holds_for_fp32_and_has_teeth(kind, lr, betas, eps, wd, clip):
    sizes = [257, 8192 + 100]
    ps = G.optim_random_tensors(sizes, 3, 0)
    ms = [np.zeros(n, f32) for n in sizes]
    vs = [np.zeros(n, f32) for n in sizes]
    worst = 0.0
    for t in range(1, 9):
        gs = G.optim_random_tensors(sizes, 4, t, scale=0.1)
        coef = G.clip(gs, clip)[1] if clip else None
        for i in range(len(sizes)):
            o = G.optim_step(kind, ps[i], gs[i], ms[i], vs[i], t, lr, betas, eps, wd, coef)
            p1, m1, v1 = _optim_f32(kind, ps[i], gs[i], ms[i], vs[i], t, lr, betas, eps, wd, coef)
            r = max(G.ratio(p1, o["p"], o["bp"]), G.ratio(m1, o["m"], o["bm"]), G.ratio(v1, o["v"], o["bv"]))
            assert r <= 1.0, (kind, t, i, r)
            worst = max(worst, r)
            # a lost tail chunk (elements past the last full 8192 left as they were) and a step taken with the
            # neighbouring element's gradient both leave the bound
            tail = o["p"].copy()
            tail[sizes[i] // 8192 * 8192:] = ps[i][sizes[i] // 8192 * 8192:]
            assert _exceeds(tail, o["p"], o["bp"])
            o2 = G.optim_step(kind, ps[i], np.roll(gs[i], 1), ms[i], vs[i], t, lr, betas, eps, wd, coef)
            assert _exceeds(o2["p"], o["p"], o["bp"]) and _exceeds(o2["v"], o["v"], o["bv"])
            if t > 1 and kind == "adam":  # bias correction taken at the wrong step count
                o3 = G.optim_step(kind, ps[i], gs[i], ms[i], vs[i], t + 1, lr, betas, eps, wd, coef)
                assert _exceeds(o3["p"], o["p"], o["bp"])
            ps[i], ms[i], vs[i] = p1, m1, v1
    assert worst > 1e-2, worst  # the bound is within two orders of what plain fp32 does


def test_optim_exact_case_is_exact():
    sizes = [1, 257, 8193]
    for kind, betas, t0 in (("adam", (0.5, 0.75), 0), ("radam", (0.5, 0.75), 0), ("radam", (0.5, 0.9375), 5)):
        rng = np.random.default_rng(7)
        ms = [G.ints(rng, n, 8, 2.0 ** -6) if t0 else np.zeros(n, f32) for n in sizes]
        vs = [np.abs(G.ints(rng, n, 16, 2.0 ** -8)) if t0 else np.zeros(n, f32) for n in sizes]
        ps = [G.ints(rng, n, 32, 2.0 ** -4) for n in sizes]
        modes = []
        for t in range(t0 + 1, t0 + (3 if t0 else 4)):
            gs = G.optim_exact_tensors(sizes, 11, t)
            norm, c = G.clip(gs, 1e9, exact=True)
            assert c == f32(1.0)
            for i in range(len(sizes)):
                o = G.optim_step(kind, ps[i], gs[i], ms[i], vs[i], t, 2.0 ** -10, betas, 2.0 ** -20, 0.0, exact_state=True)
                ms[i], vs[i] = o["m"].astype(f32), o["v"].astype(f32)
                ps[i] = o["p"].astype(f32)
                modes.append(o["mode"])
        assert set(modes) == ({0} if kind == "adam" else ({1} if t0 else {2}))
    with pytest.raises(AssertionError, match="exactness"):
        G.optim_step("adam", ps[1], G.optim_random_tensors([257], 1, 1)[0], ms[1], vs[1], 1, 1e-3, (0.5, 0.75), 1e-8, exact_state=True)
    with pytest.raises(AssertionError, match="exactness"):
        G.clip([np.full(8192, 4097.0, f32)], 1.0, exact=True)


def test_clip_matches_ref_optim():
    gs = G.optim_random_tensors([300, 9000], 5, 1)
    norm, c = G.clip(gs, 3.0)
    rn, rc = ref_optim.clip_coef([torch.from_numpy(g) for g in gs], 3.0)
    assert abs(float(norm) - float(rn)) <= 1e-6 * float(rn) and abs(float(c) - float(rc)) <= 1e-7
    assert G.clip(gs, 1e6)[1] == f32(1.0) and G.clip(gs, 0)[1] == f32(1.0) and G.clip(gs, None)[1] == f32(1.0)


# ---------------------------------------------------------------------------------------------------- TADE glue, exact
@pytest.mark.parametrize("scale", [1, 2, 3, 5, 8])
def test_tade_exact_references_match_torch(scale):
    rng = np.random.default_rng(scale)
    B, C, t = 2, 5, 12
    xn = G.ints(rng, (B, C, t), 8, 0.125)
    cg = G.ints(rng, (B, 2 * C, t * scale), 8, 0.125)
    gy = G.ints(rng, (B, C, t * scale), 8, 0.25)
    xt, ct, gt = _t(xn).requires_grad_(), _t(cg).requires_grad_(), _t(gy)
    up = F.interpolate(xt, scale_factor=scale, mode="nearest")
    y = ct[:, :C] * up + ct[:, C:]
    y.backward(gt)
    assert np.array_equal(G.upsample_nearest(xn, scale), up.detach().numpy().astype(f32))
    assert np.array_equal(G.tade_combine_exact(cg, xn, scale), y.detach().numpy().astype(f32))
    gcg, gxn = G.tade_combine_backward_exact(cg, xn, gy, scale)
    assert np.array_equal(gcg, ct.grad.numpy().astype(f32)) and np.array_equal(gxn, xt.grad.numpy().astype(f32))
    xt.grad = None
    F.interpolate(xt, scale_factor=scale, mode="nearest").backward(gt)
    assert np.array_equal(G.upsample_nearest_backward_exact(gy, scale), xt.grad.numpy().astype(f32))
    assert np.array_equal(G.leaky_relu_exact(xn, 0.25), F.leaky_relu(_t(xn), 0.25).numpy().astype(f32))
    if scale > 1:  # o / scale replaced by o % t_in, the halves of cg swapped
        wrong = np.take(xn, np.arange(t * scale) % t, axis=-1)
        assert not np.array_equal(wrong, G.upsample_nearest(xn, scale))
    sw = np.concatenate([cg[:, C:], cg[:, :C]], 1)
    assert not np.array_equal(G.tade_combine_exact(sw, xn, scale), G.tade_combine_exact(cg, xn, scale))
    with pytest.raises(AssertionError, match="exactness"):
        G.tade_combine_exact(rng.standard_normal(cg.shape).astype(f32), rng.standard_normal(xn.shape).astype(f32), scale)
    with pytest.raises(AssertionError, match="exactness"):
        G.leaky_relu_exact(xn, 0.2)


# ---------------------------------------------------------------------------------------------------- InstanceNorm1d
def _in_f32(x, eps, slope):
    x = np.asarray(x, f32)
    a = np.where(x > 0, x, x * f32(slope)).astype(f32)
    t = f32(x.shape[-1])
    mean = a.sum(-1, keepdims=True, dtype=f32) / t
    d = a - mean
    rstd = f32(1) / np.sqrt((d * d).sum(-1, keepdims=True, dtype=f32) / t + f32(eps))
    return d * rstd, rstd, a


def _in_bwd_f32(x, gy, eps, slope):
    yh, rstd, _ = _in_f32(x, eps, slope)
    gy = np.asarray(gy, f32)
    t = f32(gy.shape[-1])
    m1 = gy.sum(-1, keepdims=True, dtype=f32) / t
    m2 = (gy * yh).sum(-1, keepdims=True, dtype=f32) / t
    return rstd * (gy - m1 - yh * m2) * np.where(np.asarray(x) > 0, f32(1), f32(slope))


def test_instance_norm_reference_and_bound():
    worst = [0.0, 0.0]
    for i, (rows, t, slope, eps, kind) in enumerate(G.INSTANCE_CASES):
        x = G.instance_rows(kind, rows, t, 100 + i)
        gy = np.random.default_rng(200 + i).standard_normal((rows, t)).astype(f32)
        y, by = G.instance_norm(x, eps, slope)
        gx, bg = G.instance_norm_backward(x, gy, eps, slope)
        if t > 1 and not (kind == "const" or eps == 0):
            xt = _t(x).requires_grad_()
            yt = F.instance_norm(F.leaky_relu(xt, float(f32(slope)))[None], eps=float(f32(eps)))[0]
            yt.backward(_t(gy))
            np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(gx, xt.grad.numpy(), rtol=1e-7, atol=1e-9)
        if kind == "const":
            assert not y.any() and np.isfinite(gx).all()
        r1, r2 = G.ratio(_in_f32(x, eps, slope)[0], y, by), G.ratio(_in_bwd_f32(x, gy, eps, slope), gx, bg)
        assert r1 <= 1.0 and r2 <= 1.0, (rows, t, kind, r1, r2)
        worst = [max(worst[0], r1), max(worst[1], r2)]
    assert worst[0] > 1e-2 and worst[1] > 1e-2, worst


@pytest.mark.parametrize("mutation", ["unbiased", "eps_outside", "mean_t_minus_1", "lrelu_after", "one_pass"])
def test_instance_norm_mutations_leave_the_bound(mutation):
    caught = []
    for i, (rows, t, slope, eps, kind) in enumerate(G.INSTANCE_CASES):
        x = G.instance_rows(kind, rows, t, 100 + i).astype(np.float64)
        y, by = G.instance_norm(x, eps, slope)
        a = G.lrelu(x, slope)
        mean = a.mean(-1, keepdims=True)
        var = a.var(-1, keepdims=True)
        e = float(f32(eps))
        with np.errstate(all="ignore"):
            if mutation == "unbiased":
                mut = (a - mean) / np.sqrt(a.var(-1, keepdims=True, ddof=1 if t > 1 else 0) + e)
            elif mutation == "eps_outside":
                mut = (a - mean) / (np.sqrt(var) + e)
            elif mutation == "mean_t_minus_1":
                mm = a.sum(-1, keepdims=True) / max(t - 1, 1)
                mut = (a - mm) / np.sqrt(((a - mm) ** 2).mean(-1, keepdims=True) + e)
            elif mutation == "lrelu_after":
                mut = G.lrelu((x - x.mean(-1, keepdims=True)) / np.sqrt(x.var(-1, keepdims=True) + e), slope)
            else:  # E[a^2] - E[a]^2 in fp32
                a32 = a.astype(f32)
                m32 = a32.mean(-1, keepdims=True, dtype=f32)
                v32 = np.maximum((a32 * a32).mean(-1, keepdims=True, dtype=f32) - m32 * m32, 0)
                mut = (a32 - m32) / np.sqrt(v32 + f32(eps))
        if _exceeds(np.nan_to_num(mut, nan=1e30), y, by):
            caught.append((t, slope, kind))
    assert caught, mutation
    if mutation == "one_pass":
        assert any(k == "offset" for _, _, k in caught)
    if mutation == "eps_outside":
        assert any(k == "tiny" for _, _, k in caught)
    if mutation == "lrelu_after":
        assert all(s != 1.0 for _, s, _ in caught) and len(caught) >= 3


# ---------------------------------------------------------------------------------------------------- TADE gate
def _tade_gate_f32(x, res, scale, softmax):
    x = np.asarray(x, f32)
    C = x.shape[1] // 2
    xa = x[:, :C]
    with np.errstate(over="ignore"):
        if softmax:
            e = np.exp(xa - xa.max(1, keepdims=True))
            g = e * (f32(1) / e.sum(1, keepdims=True, dtype=f32))
        else:
            g = f32(1) / (f32(1) + np.exp(-xa))
    v = g * np.tanh(x[:, C:])
    return v + G.upsample_nearest(res, scale) if res is not None else v


def _small_gate_cases():
    for i, (B, C, T, scale, softmax, residual, kind) in enumerate(G.TADE_GATE_CASES):
        yield i, B, C, min(T, 240 // scale * scale), scale, softmax, residual, kind


def test_tade_gate_reference_and_bound():
    worst = 0.0
    for i, B, C, T, scale, softmax, residual, kind in _small_gate_cases():
        x = G.gate_logits(kind, B, C, T, 300 + i)
        res = G.ints(np.random.default_rng(i), (B, C, T // scale), 8, 0.25) if residual else None
        gy = np.random.default_rng(400 + i).standard_normal((B, C, T)).astype(f32)
        y, by = G.tade_gate(x, res, scale, softmax)
        gx, bg = G.tade_gate_backward(x, gy, softmax)
        xt = _t(x).requires_grad_()
        gt = torch.softmax(xt[:, :C], 1) if softmax else torch.sigmoid(xt[:, :C])
        yt = gt * torch.tanh(xt[:, C:])
        if res is not None:
            yt = yt + F.interpolate(_t(res), scale_factor=scale, mode="nearest")
        yt.backward(_t(gy))
        np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(gx, xt.grad.numpy(), rtol=1e-9, atol=1e-15)
        r = G.ratio(_tade_gate_f32(x, res, scale, softmax), y, by)
        assert r <= 1.0, (i, r)
        worst = max(worst, r)
        if kind == "one":  # tanh saturated at 1: the outputs are the softmax itself and sum to 1 per column
            assert np.all(np.abs(y.sum(1) - 1.0) <= 1e-12)
    assert worst > 1e-2, worst


@pytest.mark.parametrize("mutation", ["softmax_over_time", "residual_unscaled", "no_dot", "no_max"])
def test_tade_gate_mutations_leave_the_bound(mutation):
    caught = 0
    for i, B, C, T, scale, softmax, residual, kind in _small_gate_cases():
        x = G.gate_logits(kind, B, C, T, 300 + i).astype(np.float64)
        res = G.ints(np.random.default_rng(i), (B, C, T // scale), 8, 0.25) if residual else None
        gy = np.random.default_rng(400 + i).standard_normal((B, C, T))
        y, by = G.tade_gate(x, res, scale, softmax)
        gx, bg = G.tade_gate_backward(x, gy, softmax)
        th = np.tanh(x[:, C:])
        if mutation == "softmax_over_time" and softmax:
            e = np.exp(x[:, :C] - x[:, :C].max(2, keepdims=True))
            mut = e / e.sum(2, keepdims=True) * th + (G.upsample_nearest(res, scale) if residual else 0)
            caught += _exceeds(mut, y, by)
        elif mutation == "residual_unscaled" and residual and scale > 1:
            idx = np.minimum(np.arange(T), T // scale - 1)
            mut = y - G.upsample_nearest(res, scale) + np.take(res, idx, axis=-1)
            caught += _exceeds(mut, y, by)
        elif mutation == "no_dot" and softmax and C > 1:
            g = G._softmax_gate(x[:, :C])[0]
            mut = np.concatenate([g * gy * th, gx[:, C:]], 1)
            caught += _exceeds(mut, gx, bg)
        elif mutation == "no_max" and softmax and kind == "spread":
            with np.errstate(all="ignore"):
                e = np.exp(x[:, :C]).astype(f32)  # overflows in fp32 without the max subtraction
                mut = np.nan_to_num((e / e.sum(1, keepdims=True)).astype(np.float64) * th, nan=1e30) + (G.upsample_nearest(res, scale) if residual else 0)
            caught += _exceeds(mut, y, by)
    assert caught >= 2, mutation


# ---------------------------------------------------------------------------------------------------- LayerNorm
def _ln_f32(x, gamma, beta, eps):
    x = np.asarray(x, f32)
    C = f32(x.shape[1])
    mean = x.sum(1, keepdims=True, dtype=f32) / C
    d = x - mean
    rstd = f32(1) / np.sqrt((d * d).sum(1, keepdims=True, dtype=f32) / C + f32(eps))
    return d * rstd * gamma.reshape(1, -1, 1) + beta.reshape(1, -1, 1), mean[:, 0], rstd[:, 0]


def _ln_bwd_f32(x, gy, gamma, mean, rstd):
    x, gy = np.asarray(x, f32), np.asarray(gy, f32)
    C = f32(x.shape[1])
    xh = (x - mean[:, None]) * rstd[:, None]
    gg = gy * gamma.reshape(1, -1, 1)
    m1 = gg.sum(1, keepdims=True, dtype=f32) / C
    m2 = (gg * xh).sum(1, keepdims=True, dtype=f32) / C
    return rstd[:, None] * (gg - m1 - xh * m2), (gy * xh).sum((0, 2), dtype=f32), gy.sum((0, 2), dtype=f32)


def test_layernorm_reference_and_bound():
    worst = 0.0
    for i, (B, C, T, eps, kind) in enumerate(G.LAYERNORM_CASES):
        x, gamma, beta, gy = G.layernorm_data(B, C, T, kind, 500 + i)
        o = G.channel_layernorm(x, gamma, beta, eps)
        y32, m32, r32 = _ln_f32(x, gamma, beta, eps)
        if C > 1:
            xt, gt, bt = _t(x).requires_grad_(), _t(gamma).requires_grad_(), _t(beta).requires_grad_()
            yt = F.layer_norm(xt.transpose(1, 2), (C,), gt, bt, float(f32(eps))).transpose(1, 2)
            yt.backward(_t(gy))
            np.testing.assert_allclose(o["y"], yt.detach().numpy(), rtol=1e-7, atol=1e-9)
            # backward reference from the float64 statistics rounded to fp32 equals autograd within that rounding
            b = G.channel_layernorm_backward(x, gy, gamma, o["mean"].astype(f32), o["rstd"].astype(f32))
            np.testing.assert_allclose(b["dx"], xt.grad.numpy(), rtol=1e-4, atol=1e-4 * np.abs(xt.grad.numpy()).max())
            np.testing.assert_allclose(b["dbeta"], bt.grad.numpy(), rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(b["dgamma"], gt.grad.numpy(), rtol=1e-4, atol=1e-4 * (np.abs(gt.grad.numpy()).max() + 1))
        rs = [G.ratio(y32, o["y"], o["by"]), G.ratio(m32, o["mean"], o["bmean"]), G.ratio(r32, o["rstd"], o["brstd"])]
        b = G.channel_layernorm_backward(x, gy, gamma, m32, r32)
        dx32, dg32, db32 = _ln_bwd_f32(x, gy, gamma, m32, r32)
        rs += [G.ratio(dx32, b["dx"], b["bdx"]), G.ratio(dg32, b["dgamma"], b["bdgamma"]), G.ratio(db32, b["dbeta"], b["bdbeta"])]
        assert max(rs) <= 1.0, (B, C, T, kind, rs)
        worst = max(worst, max(rs[:4]))
    assert worst > 1e-2, worst


@pytest.mark.parametrize("mutation", ["c_minus_1", "eps_outside", "stale_frame", "last_block_dropped"])
def test_layernorm_mutations_leave_the_bound(mutation):
    caught = 0
    for i, (B, C, T, eps, kind) in enumerate(G.LAYERNORM_CASES):
        x, gamma, beta, gy = G.layernorm_data(B, C, T, kind, 500 + i)
        o = G.channel_layernorm(x, gamma, beta, eps)
        xd = x.astype(np.float64)
        c = xd - xd.mean(1, keepdims=True)
        g3, b3 = gamma.reshape(1, -1, 1), beta.reshape(1, -1, 1)
        m32, r32 = o["mean"].astype(f32), o["rstd"].astype(f32)
        b = G.channel_layernorm_backward(x, gy, gamma, m32, r32)
        tg = gy.astype(np.float64) * ((xd - m32[:, None]) * r32[:, None])
        with np.errstate(all="ignore"):
            if mutation == "c_minus_1" and C > 1 and kind != "gamma0":
                mut = c / np.sqrt(xd.var(1, keepdims=True, ddof=1) + eps) * g3 + b3
                caught += _exceeds(mut, o["y"], o["by"])
            elif mutation == "eps_outside" and eps == 1e-5 and kind == "offset":
                mut = c / (np.sqrt(xd.var(1, keepdims=True)) + eps) * g3 + b3
                caught += _exceeds(mut, o["y"], o["by"])
            elif mutation == "stale_frame" and T % 32:  # an inactive lane of the last block adds one more frame
                caught += _exceeds(b["dgamma"] + tg[-1, :, 0], b["dgamma"], b["bdgamma"]) and \
                    _exceeds(b["dbeta"] + gy[-1, :, 0], b["dbeta"], b["bdbeta"])
            elif mutation == "last_block_dropped" and T > 1:
                lo = (T - 1) // 32 * 32
                caught += _exceeds(b["dgamma"] - tg[-1, :, lo:].sum(-1), b["dgamma"], b["bdgamma"]) and \
                    _exceeds(b["dbeta"] - gy[-1, :, lo:].astype(np.float64).sum(-1), b["dbeta"], b["bdbeta"])
    assert caught >= 1, mutation


def test_layernorm_param_grads_exact_data():
    rng = np.random.default_rng(9)
    B, C, T = 3, 9, 1000
    x, gy = G.ints(rng, (B, C, T), 8, 0.125), G.ints(rng, (B, C, T), 8, 0.25)
    mean, rstd = G.ints(rng, (B, T), 4, 0.5), np.exp2(rng.integers(-2, 3, (B, T))).astype(f32)
    dg, db = G.channel_layernorm_param_grads_exact(x, gy, mean, rstd)
    xh = (x.astype(np.float64) - mean[:, None]) * rstd[:, None]
    assert np.array_equal(dg, (gy * xh).sum((0, 2)).astype(f32)) and np.array_equal(db, gy.astype(np.float64).sum((0, 2)).astype(f32))
    for perm in range(3):  # fp32 sums in shuffled orders reproduce it
        p = np.random.default_rng(perm).permutation(B * T)
        terms = (gy * xh).transpose(1, 0, 2).reshape(C, -1)[:, p].astype(f32)
        assert np.array_equal(np.add.reduce(terms, 1, dtype=f32), dg)
    with pytest.raises(AssertionError, match="exactness"):
        G.channel_layernorm_param_grads_exact(rng.standard_normal((B, C, T)), gy, mean, rstd)


# ---------------------------------------------------------------------------------------------------- WaveNet gate
def test_wavenet_gate_reference_and_bound():
    g = G.wavenet_gate_inputs(2, 3, 64, 1)
    gz = np.random.default_rng(2).standard_normal((2, 3, 64)).astype(f32)
    z, bz = G.gate(g)
    gg, bg = G.gate_backward(g, gz)
    gt = _t(g).requires_grad_()
    zt = torch.tanh(gt[:, :3]) * torch.sigmoid(gt[:, 3:])
    zt.backward(_t(gz))
    np.testing.assert_allclose(z, zt.detach().numpy(), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(gg, gt.grad.numpy(), rtol=1e-9, atol=1e-15)
    with np.errstate(over="ignore"):
        z32 = np.tanh(g[:, :3]) * (f32(1) / (f32(1) + np.exp(-g[:, 3:])))
    assert G.ratio(z32, z, bz) <= 1.0 and np.isfinite(z).all() and np.isfinite(gg).all()
    # the halves swapped, and a gradient without the (1 - sg) factor, leave the bound
    assert _exceeds(np.tanh(g[:, 3:].astype(np.float64)) / (1 + np.exp(-g[:, :3].astype(np.float64))), z, bz)
    sg = 1 / (1 + np.exp(-g[:, 3:].astype(np.float64)))
    assert _exceeds(np.concatenate([gg[:, :3], gz * np.tanh(g[:, :3].astype(np.float64)) * sg], 1), gg, bg)


# ---------------------------------------------------------------------------------------------------- loss reductions
@pytest.mark.parametrize("mode", list(G.REDUCE_MODES))
def test_reduce_reference_matches_torch(mode):
    for n in (1, 257, 2049, 300000):
        x, y, c, s = G.reduce_data(mode, n, n)
        xt = _t(x).requires_grad_()
        yt = _t(y) if y is not None else None
        ref = {"mse_const": lambda: ((xt - c) ** 2).mean(), "l1": lambda: (xt - yt).abs().mean(), "hinge": lambda: F.relu(c - s * xt).mean(),
               "linear": lambda: (s * xt).mean(), "mse": lambda: ((xt - yt) ** 2).mean()}[mode]() * 0.5
        ref.backward()
        for ws in (1, 7, 1024):
            got = G.reduce_mean_exact(mode, x, y, c, s, 0.5, ws_floats=ws)
            assert abs(float(got) - ref.item()) <= 1e-6 * abs(ref.item()) + 1e-30
        assert G.reduce_mean_exact(mode, x, y, c, s, 0.5, prev=f32(3.0)) == f32(3.0) + G.reduce_mean_exact(mode, x, y, c, s, 0.5)
        n2 = 1 << (n - 1).bit_length()
        gx = G.reduce_mean_backward_exact(mode, x, y, c, s, weight=n / n2, gout=0.5)
        np.testing.assert_allclose(gx, xt.grad.numpy() * 2 * (n / n2) * 0.5, rtol=1e-6, atol=0)
    x, y, c, s = G.reduce_data(mode, 5000, 1)
    if mode == "hinge":
        assert np.any(c - s * x == 0)
    if mode == "l1":
        assert np.any(x == y)
    # ignoring the elements past 1024 * 2048 changes the result
    n, k = 5000001, 1024 * 2048
    x, y, c, s = G.reduce_data(mode, n, 3)
    full = G.reduce_mean_exact(mode, x, y, c, s, 1.0)
    cut = f32(float(G.reduce_terms(mode, x[:k], None if y is None else y[:k], c, s)[0].sum()) / n)
    assert full != cut


def test_reduce_exactness_guard():
    with pytest.raises(AssertionError, match="exactness"):
        G.reduce_mean_exact("mse_const", np.random.default_rng(0).standard_normal(100).astype(f32), None, 1.0, 1.0)
    with pytest.raises(AssertionError, match="exactness"):
        G.reduce_mean_exact("mse_const", G.reduce_data("mse_const", 5000001, 1)[0], None, 1.0, 1.0, ws_floats=1)
    for mode in G.REDUCE_MODES:  # the data of the GPU test pass the guard at every size and workspace
        for n in G.REDUCE_SIZES[-3:]:
            x, y, c, s = G.reduce_data(mode, n, n % 1000 + len(mode))
            G.reduce_mean_exact(mode, x, y, c, s, 0.5)
            x, y, c, s = G.reduce_data(mode, n, n % 1000, coarse=True)
            for ws in (1, 7):
                G.reduce_mean_exact(mode, x, y, c, s, 1.0, ws_floats=ws)


def test_duration_loss_and_symbol_embed_references():
    rng = np.random.default_rng(4)
    x, ds = rng.standard_normal(257).astype(f32), rng.integers(0, 40, 257)
    loss, bl, gx, bg = G.duration_loss(x, ds, 1.0)
    xt = _t(x).requires_grad_()
    lt = F.mse_loss(xt, torch.log(_t(ds) + 1.0))
    lt.backward()
    assert abs(loss - lt.item()) <= 1e-12 and np.allclose(gx, xt.grad.numpy(), rtol=1e-12, atol=0)
    r = x - np.log(ds.astype(f32) + f32(1.0))
    assert abs(float((r.astype(np.float64) ** 2).mean()) - loss) <= bl
    gy = G.ints(rng, (2, 3, 50), 8, 0.25)
    idx = rng.integers(0, 7, (2, 50))
    d = G.symbol_embed_backward_exact(gy, idx, 7)
    tab = torch.zeros(7, 3, dtype=torch.float64, requires_grad=True)
    F.embedding(torch.from_numpy(idx), tab).transpose(1, 2).backward(_t(gy))
    assert np.array_equal(d, tab.grad.numpy().astype(f32))
