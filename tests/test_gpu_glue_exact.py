"""The optimizer, normalisation, gate and loss-reduction kernels element by element against oracle/glue_exact.py:
bit for bit on exact data, and within a derived per-element bound of the float64 value where the arithmetic rounds
(tests/test_glue_exact_cpu.py checks the references, that plain fp32 meets the bounds and that kernel mistakes do not).
Sizes sit on the edges of each kernel's chunking: the optimizer's 8192-element chunks, the 132 * 16 * 256 = 540,672
element stride of the tade.cu grid-stride loops, the 32-frame LayerNorm blocks, the float4 / scalar split of the gate
and the 1024 * 2048 element grid clamp of the reductions.  Output buffers start as NaN, so an unwritten element shows."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import glue_exact as G

pytestmark = pytest.mark.gpu
f32 = np.float32
STRIDE = 132 * 16 * 256  # elements one pass of a tade.cu grid-stride loop covers
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    yield torch.device("cuda:0")
    if WORST:
        print("\n[glue_exact] worst error / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


def _d(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _n(t):
    return t.detach().cpu().numpy()


def _nan(shape, dev):
    return torch.full(shape, float("nan"), device=dev, dtype=torch.float32)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _within(family, what, got, ref, bound):
    r = G.ratio(got, ref, bound)
    WORST[family] = max(WORST.get(family, 0.0), r)
    assert r <= 1.0, f"{what}: error {r:.3f} x the bound"


def _same(what, got, ref):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = ~((got == ref) | (np.isnan(got) & np.isnan(ref)))
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} elements differ, first at {np.argwhere(bad)[0].tolist()}"


def _call(name, *args):
    from parallelwavegan_b200 import capi, ops

    capi.check(getattr(capi.lib(), name)(*args, ops._stream()), name)


# ---------------------------------------------------------------------------------------------------- fused optimizer
NORM_REL = (G.CHUNK // 256 + 14) * G.U / 2 + 2 * G.U  # fp32 chunk sums of squares (depth 32 + 13), the root halves it


def _params(init, dev):
    return [torch.nn.Parameter(_d(a, dev)) for a in init]


def _state(opt, p):
    st = opt.state.get(p, {})
    if len(st) == 0:
        return np.zeros(p.numel(), f32), np.zeros(p.numel(), f32), 0
    return _n(st["exp_avg"]).reshape(-1), _n(st["exp_avg_sq"]).reshape(-1), int(st["step"])


def _step(opt, kind, params, grads, clip=None, exact=False, write=False, what=""):
    """sets the gradients (None leaves the parameter without one), takes one step and holds every tensor to the
    reference computed from its own state before the step"""
    dev = params[0].device
    live, idle = [], []
    hyper = {id(p): g for g in opt.param_groups for p in g["params"]}
    for p, g in zip(params, grads):
        if g is None:
            p.grad = None
            idle.append((p, _n(p).copy()))
        else:
            p.grad = _d(g, dev)
            live.append((p, g, _n(p).reshape(-1).copy()) + _state(opt, p))
    opt.step(max_grad_norm=clip, write_clipped_grad=write)
    coef = None
    if clip is not None and clip > 0:
        norm, c = G.clip([g for _, g, *_ in live], clip, exact=exact)
        got = _n(opt.last_grad_norm)
        if exact:
            assert got[0] == norm and got[1] == c, f"{what}: norm / coefficient {got.tolist()} != {float(norm)!r}, {float(c)!r}"
        else:
            assert abs(float(got[0]) - float(norm)) <= NORM_REL * float(norm), f"{what}: norm {got[0]} vs {norm}"
            c = f32(clip) / (got[0] + f32(1e-6))
            assert got[1] == (f32(1.0) if c > f32(1.0) else c), f"{what}: coefficient is not min(1, max_norm / (norm + 1e-6f))"
        coef = got[1]
    for i, (p, g, p0, m0, v0, t) in enumerate(live):
        h = hyper[id(p)]
        o = G.optim_step(kind, p0, g.reshape(-1), m0, v0, t + 1, h["lr"], h["betas"], h["eps"], h["weight_decay"], coef, exact_state=exact)
        m1, v1, t1 = _state(opt, p)
        assert t1 == t + 1
        tag = f"{what} tensor {i} ({p.numel()} elements) step {t + 1}"
        if exact:
            _same(tag + " exp_avg", m1, o["m"].astype(f32))
            _same(tag + " exp_avg_sq", v1, o["v"].astype(f32))
        _within("optimizer", tag + " exp_avg", m1, o["m"], o["bm"])
        _within("optimizer", tag + " exp_avg_sq", v1, o["v"], o["bv"])
        _within("optimizer", tag + " parameter", _n(p).reshape(-1), o["p"], o["bp"])
        _same(tag + " gradient", _n(p.grad).reshape(-1), G.clipped_grad(g, coef).reshape(-1) if write and coef is not None else g.reshape(-1))
    for p, p0 in idle:
        _same(what + " parameter without gradient", _n(p), p0)


def _edge_model(dev, seed=1, exact=True):
    """the chunk-edge sizes, a zero-element parameter and (index 5) a parameter that never gets a gradient"""
    sizes = G.OPTIM_EDGE_SIZES[:5] + [300] + G.OPTIM_EDGE_SIZES[5:] + [0]
    rng = np.random.default_rng(seed)
    init = [G.ints(rng, n, 32, 2.0 ** -4) if exact else rng.standard_normal(n).astype(f32) for n in sizes]
    return sizes, _params(init, dev)


def _grads(sizes, seed, t, exact, none_at=(5,), scale=1.0):
    gs = G.optim_exact_tensors(sizes, seed, t) if exact else G.optim_random_tensors(sizes, seed, t, scale)
    return [None if i in none_at else g for i, g in enumerate(gs)]


@pytest.mark.parametrize("case", ["adam", "adam_wd", "radam_unrectified", "radam_rectified"])
def test_optimizer_exact(dev, case):
    """betas (0.5, 0.75), gradients k / 64: exp_avg, exp_avg_sq, the total norm and the (non-binding) coefficient bit for
    bit; RAdam's rectified mode starts from an exact state at step 5 with beta2 = 0.9375, where n_sma >= 5 from step 6"""
    from parallelwavegan_b200 import optimizers

    sizes, ps = _edge_model(dev)
    kind = "adam" if case.startswith("adam") else "radam"
    kw = dict(lr=2.0 ** -10, betas=(0.5, 0.9375 if case == "radam_rectified" else 0.75), eps=2.0 ** -20,
              weight_decay=2.0 ** -3 if case in ("adam_wd", "radam_unrectified") else 0.0)
    opt = (optimizers.FusedAdam if kind == "adam" else optimizers.RAdam)(ps, **kw)
    t0 = 0
    if case == "radam_rectified":
        t0 = 5
        rng = np.random.default_rng(3)
        for i, p in enumerate(ps):
            if i != 5:
                opt.state[p] = dict(step=5, exp_avg=_d(G.ints(rng, p.numel(), 8, 2.0 ** -6), dev),
                                    exp_avg_sq=_d(np.abs(G.ints(rng, p.numel(), 16, 2.0 ** -8)), dev))
    steps = {"adam": 3, "adam_wd": 1, "radam_unrectified": 3, "radam_rectified": 2}[case]
    for t in range(t0 + 1, t0 + steps + 1):
        assert G.radam_mode(t, kw["betas"])[0] == (1 if case == "radam_rectified" else 2)
        _step(opt, kind, ps, _grads(sizes, 21, t, True), clip=1e9, exact=True, what=case)


@pytest.mark.parametrize("kind,lr,betas,eps,wd,clip,big", [
    ("adam", 2e-4, (0.5, 0.9), 1e-8, 0.0, None, False), ("adam", 2e-4, (0.5, 0.9), 1e-8, 0.01, 3.0, True),
    ("radam", 1e-4, (0.9, 0.999), 1e-6, 0.0, 10.0, True), ("radam", 1e-4, (0.9, 0.999), 1e-6, 0.01, None, False)])
def test_optimizer_recipe(dev, kind, lr, betas, eps, wd, clip, big):
    """random data, the recipe hyper-parameters, 7 steps (RAdam's rectification switches on at step 6); ``big`` is a model
    of 320 tensors, so the chunk table has several hundred rows and every tensor has its own data"""
    from parallelwavegan_b200 import optimizers

    if big:
        sizes = G.optim_big_sizes()
        ps = _params(G.optim_random_tensors(sizes, 30, 0), dev)
        none_at = (7,)
    else:
        sizes, ps = _edge_model(dev, exact=False)
        none_at = (5,)
    opt = (optimizers.FusedAdam if kind == "adam" else optimizers.RAdam)(ps, lr=lr, betas=betas, eps=eps, weight_decay=wd)
    for t in range(1, 8):
        _step(opt, kind, ps, _grads(sizes, 31, t, False, none_at, scale=0.05), clip=clip, write=(t % 2 == 0), what=f"{kind} big={big}")
    assert len(opt._tables) <= 8


def test_optimizer_clip_semantics(dev):
    from parallelwavegan_b200 import optimizers

    sizes = [257, 8193, 40]
    init = G.optim_random_tensors(sizes, 40, 0)
    gs = G.optim_random_tensors(sizes, 41, 1)

    def fresh(groups=False):
        ps = _params(init, dev)
        arg = [dict(params=ps[:2], lr=1e-3), dict(params=ps[2:], lr=5e-2)] if groups else ps
        return ps, optimizers.FusedAdam(arg, lr=1e-3, betas=(0.5, 0.9))

    # a clip that does not bind, None and 0 all give the unclipped step; only the first records a norm
    base, ob = fresh()
    _step(ob, "adam", base, gs, what="unclipped")
    assert ob.last_grad_norm is None
    for clip in (1e6, None, 0):
        ps, o = fresh()
        _step(o, "adam", ps, gs, clip=clip, write=True, what=f"clip {clip}")
        for a, b in zip(ps, base):
            assert torch.equal(a.detach(), b.detach())
        if clip:
            assert float(o.last_grad_norm[1]) == 1.0
        else:
            assert o.last_grad_norm is None
    # two groups with different lr share one global norm; the clipped gradients are written back only when asked
    for write in (True, False):
        ps, o = fresh(groups=True)
        _step(o, "adam", ps, gs, clip=0.5, write=write, what=f"two groups write={write}")
        norm = G.clip(gs, 0.5)[0]
        assert abs(float(o.last_grad_norm[0]) - float(norm)) <= NORM_REL * float(norm) and float(o.last_grad_norm[1]) < 0.1


def test_optimizer_host_tables(dev):
    """re-allocated gradients, a parameter that gains a gradient later (two step-count buckets), more distinct parameter
    subsets than the table cache holds, and a step whose only gradient belongs to an empty parameter"""
    from parallelwavegan_b200 import optimizers

    sizes = [1, 8193, 300, 0, 8192, 77, 2 * 8192 + 1, 255, 4096, 31]

    def run():
        ps = _params(G.optim_random_tensors(sizes, 50, 0), dev)
        o = optimizers.RAdam(ps, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01)
        keep = []
        for t in range(1, 13):
            gs = G.optim_random_tensors(sizes, 51, t)
            if t <= 2:
                gs[2] = None  # tensor 2 gains its gradient at step 3: from then on two buckets
            elif t >= 4:
                gs[(t - 4) % len(sizes)] = None  # a different subset every step: 9 more table keys
                gs[(t - 3) % len(sizes)] = None
            _step(o, "radam", ps, gs, clip=5.0 if t % 3 else None, what=f"host tables step {t}")
            keep.append([p.grad for p in ps])  # the old gradients stay alive, so the new ones get new addresses
            o.zero_grad(set_to_none=True)
        gs = [None] * len(sizes)
        gs[3] = np.zeros(0, f32)
        _step(o, "radam", ps, gs, clip=1.0, what="only the empty parameter")
        assert _n(o.last_grad_norm).tolist() == [0.0, 1.0]
        return ps

    a, b = run(), run()
    for x, y in zip(a, b):
        assert torch.equal(x.detach(), y.detach())


# ---------------------------------------------------------------------------------------------------- TADE glue, exact
@pytest.mark.parametrize("B,Cc,t_in,scale", [
    (2, 1, 13, 1), (2, 5, 13, 2), (2, 64, 9, 3), (1, 5, 11, 4), (3, 1, 7, 5), (1, 64, 10, 8), (2, 64, 1408, 4), (2, 64, 5632, 2),
    (1, 1, STRIDE - 1, 1), (1, 1, STRIDE + 1, 1), (1, 5, (2 * STRIDE + 5) // 5, 3)])
def test_tade_glue_exact(dev, B, Cc, t_in, scale):
    from parallelwavegan_b200 import ops

    rng = np.random.default_rng([B, Cc, t_in, scale])
    t_out = t_in * scale
    xn = G.ints(rng, (B, Cc, t_in), 8, 0.125)
    cg = G.ints(rng, (B, 2 * Cc, t_out), 8, 0.125)
    gy = G.ints(rng, (B, Cc, t_out), 8, 0.25)
    xd, cd, gd = _d(xn, dev), _d(cg, dev), _d(gy, dev)
    y = _nan((B, Cc, t_out), dev)
    _call("pwgb_upsample_nearest_forward", _p(xd), _p(y), B * Cc, t_in, scale)
    _same("upsample_nearest", _n(y), G.upsample_nearest(xn, scale))
    gx = _nan((B, Cc, t_in), dev)
    _call("pwgb_upsample_nearest_backward", _p(gd), _p(gx), B * Cc, t_in, scale)
    _same("upsample_nearest_backward", _n(gx), G.upsample_nearest_backward_exact(gy, scale))
    y = _nan(tuple(cg.shape), dev)
    _call("pwgb_leaky_relu_forward", _p(cd), _p(y), cd.numel(), 0.25)
    _same("leaky_relu", _n(y), G.leaky_relu_exact(cg, 0.25))
    y = _nan((B, Cc, t_out), dev)
    _call("pwgb_tade_combine_forward", _p(cd), _p(xd), _p(y), B, Cc, t_out, scale)
    _same("tade_combine", _n(y), G.tade_combine_exact(cg, xn, scale))
    if scale > 1 and t_in < 100:  # the wrappers reach the same kernels
        _same("ops.tade_combine", _n(ops.tade_combine(cd, xd, scale)), _n(y))
        _same("ops.upsample_nearest", _n(ops.upsample_nearest(xd, scale)), G.upsample_nearest(xn, scale))
    gcg, gxn = _nan(tuple(cg.shape), dev), _nan(tuple(xn.shape), dev)
    _call("pwgb_tade_combine_backward", _p(cd), _p(xd), _p(gd), _p(gcg), _p(gxn), B, Cc, t_out, scale)
    rcg, rxn = G.tade_combine_backward_exact(cg, xn, gy, scale)
    _same("tade_combine_backward gcg", _n(gcg), rcg)
    _same("tade_combine_backward gxn", _n(gxn), rxn)


# ---------------------------------------------------------------------------------------------------- InstanceNorm1d
def _instance(dev, x, gy, eps, slope):
    rows, t = x.shape
    xd, gd = _d(x, dev), _d(gy, dev)
    y, gx = _nan((rows, t), dev), _nan((rows, t), dev)
    _call("pwgb_instance_norm_forward", _p(xd), _p(y), rows, t, float(eps), float(slope))
    _call("pwgb_instance_norm_backward", _p(xd), _p(gd), _p(gx), rows, t, float(eps), float(slope))
    return _n(y), _n(gx)


@pytest.mark.parametrize("case", range(len(G.INSTANCE_CASES)))
def test_instance_norm(dev, case):
    rows, t, slope, eps, kind = G.INSTANCE_CASES[case]
    x = G.instance_rows(kind, rows, t, 100 + case)
    gy = np.random.default_rng(200 + case).standard_normal((rows, t)).astype(f32)
    y, gx = _instance(dev, x, gy, eps, slope)
    ry, by = G.instance_norm(x, eps, slope)
    rg, bg = G.instance_norm_backward(x, gy, eps, slope)
    what = f"instance_norm rows {rows} t {t} slope {slope} {kind}"
    if kind == "const":
        assert not y.any() and np.isfinite(gx).all(), what
    _within("instance_norm", what, y, ry, by)
    _within("instance_norm_backward", what + " backward", gx, rg, bg)
    y2, gx2 = _instance(dev, x, gy, eps, slope)
    _same(what + " second run", y2, y)
    _same(what + " backward second run", gx2, gx)


def test_instance_norm_many_rows(dev):
    """more rows than a grid's y or z extent holds: the launch indexes rows by grid.x alone"""
    rows, t = 70000, 8
    x = G.instance_rows("plain", rows, t, 7)
    gy = np.random.default_rng(8).standard_normal((rows, t)).astype(f32)
    y, gx = _instance(dev, x, gy, 1e-5, 0.2)
    _within("instance_norm", "70000 rows", y, *G.instance_norm(x, 1e-5, 0.2))
    _within("instance_norm_backward", "70000 rows backward", gx, *G.instance_norm_backward(x, gy, 1e-5, 0.2))


# ---------------------------------------------------------------------------------------------------- TADE gate
@pytest.mark.parametrize("case", range(len(G.TADE_GATE_CASES)))
def test_tade_gate(dev, case):
    from parallelwavegan_b200 import ops

    B, Cc, T, scale, softmax, residual, kind = G.TADE_GATE_CASES[case]
    x = G.gate_logits(kind, B, Cc, T, 300 + case)
    res = G.ints(np.random.default_rng(case), (B, Cc, T // scale), 8, 0.25) if residual else None
    gy = np.random.default_rng(400 + case).standard_normal((B, Cc, T)).astype(f32)
    xd = _d(x, dev)
    rd = _d(res, dev) if residual else None
    yd = _nan((B, Cc, T), dev)
    _call("pwgb_tade_gate_forward", _p(xd), _p(rd), _p(yd), B, Cc, T, scale, int(softmax))
    y = _n(yd)
    if T < 1000:
        _same("ops.tade_gate", _n(ops.tade_gate(xd, rd, scale, "softmax" if softmax else "sigmoid")), y)
    gx, gd = _nan(tuple(x.shape), dev), _d(gy, dev)
    _call("pwgb_tade_gate_backward", _p(xd), _p(gd), _p(gx), B, Cc, T, int(softmax))
    ry, by = G.tade_gate(x, res, scale, softmax)
    rg, bg = G.tade_gate_backward(x, gy, softmax)
    what = f"tade_gate {G.TADE_GATE_CASES[case]}"
    assert np.isfinite(y).all() and np.isfinite(_n(gx)).all(), what
    _within("tade_gate", what, y, ry, by)
    _within("tade_gate_backward", what + " backward", _n(gx), rg, bg)
    if kind == "one":  # tanh is exactly 1: the outputs are the softmax, and each column sums to 1 within the bounds
        assert np.all(np.abs(y.astype(np.float64).sum(1) - 1.0) <= by.sum(1) + Cc * G.U), what


# ---------------------------------------------------------------------------------------------------- channel LayerNorm
def _layernorm_backward(dev, x, gy, gamma, mean, rstd):
    from parallelwavegan_b200 import capi

    B, Cc, T = x.shape
    dx, dg, db = _nan((B, Cc, T), dev), _nan((Cc,), dev), _nan((Cc,), dev)
    nbytes = capi.lib().pwgb_channel_layernorm_backward_workspace(B, Cc, T)
    ws = _nan(((nbytes + 3) // 4,), dev)
    ins = [_d(a, dev) for a in (x, gy, gamma, mean, rstd)]  # held until the call has been enqueued
    _call("pwgb_channel_layernorm_backward", *[_p(a) for a in ins], B, Cc, T, _p(dx), _p(dg), _p(db), _p(ws), C.c_size_t(nbytes))
    return _n(dx), _n(dg), _n(db)


@pytest.mark.parametrize("case", range(len(G.LAYERNORM_CASES)))
def test_channel_layernorm(dev, case):
    from parallelwavegan_b200 import ops

    B, Cc, T, eps, kind = G.LAYERNORM_CASES[case]
    x, gamma, beta, gy = G.layernorm_data(B, Cc, T, kind, 500 + case)
    y, mean, rstd = (_n(t) for t in ops.channel_layer_norm_raw(_d(x, dev), _d(gamma, dev), _d(beta, dev), eps, stats=True))
    o = G.channel_layernorm(x, gamma, beta, eps)
    what = f"channel_layernorm {G.LAYERNORM_CASES[case]}"
    _within("layernorm", what + " y", y, o["y"], o["by"])
    _within("layernorm", what + " mean", mean, o["mean"], o["bmean"])
    _within("layernorm", what + " rstd", rstd, o["rstd"], o["brstd"])
    if kind == "gamma0":
        _same(what + " y with gamma 0", y, np.broadcast_to(beta.reshape(1, -1, 1), y.shape))
    dx, dg, db = _layernorm_backward(dev, x, gy, gamma, mean, rstd)
    b = G.channel_layernorm_backward(x, gy, gamma, mean, rstd)
    _within("layernorm_backward", what + " dx", dx, b["dx"], b["bdx"])
    _within("layernorm_param_grads", what + " dgamma", dg, b["dgamma"], b["bdgamma"])
    _within("layernorm_param_grads", what + " dbeta", db, b["dbeta"], b["bdbeta"])
    again = _layernorm_backward(dev, x, gy, gamma, mean, rstd)
    for n, u, v in zip(("dx", "dgamma", "dbeta"), again, (dx, dg, db)):
        _same(what + f" {n} second run", u, v)


@pytest.mark.parametrize("B,Cc,T", [(3, 9, 1000), (1, 7, 31), (1, 64, 33), (3, 384, 1), (1, 8, 5000)])
def test_channel_layernorm_param_grads_exact(dev, B, Cc, T):
    """with the statistics given as exact numbers (mean k / 2, rstd a power of two) dgamma and dbeta are sums of exact
    products: bit for bit, whatever the order of the block partials and with the last block's inactive lanes at zero"""
    rng = np.random.default_rng([B, Cc, T])
    x, gy = G.ints(rng, (B, Cc, T), 8, 0.125), G.ints(rng, (B, Cc, T), 8, 0.25)
    mean, rstd = G.ints(rng, (B, T), 4, 0.5), np.exp2(rng.integers(-2, 3, (B, T))).astype(f32)
    _, dg, db = _layernorm_backward(dev, x, gy, np.ones(Cc, f32), mean, rstd)
    rg, rb = G.channel_layernorm_param_grads_exact(x, gy, mean, rstd)
    _same("dgamma", dg, rg)
    _same("dbeta", db, rb)


# ---------------------------------------------------------------------------------------------------- WaveNet gate
def _gate(dev, g, gz, off=0):
    B, H2, T = g.shape
    H = H2 // 2

    def at(a):
        buf = torch.zeros(a.size + off, device=dev)
        v = buf[off:].view(a.shape)
        v.copy_(_d(a, dev))
        return v

    gd, gzd = at(g), at(gz)
    z, gg = at(np.full((B, H, T), np.nan, f32)), at(np.full((B, H2, T), np.nan, f32))
    _call("pwgb_gate_forward", _p(gd), _p(z), B, H, T)
    _call("pwgb_gate_backward", _p(gd), _p(gzd), _p(gg), B, H, T)
    return _n(z), _n(gg)


@pytest.mark.parametrize("B,H,T", [(2, 1, 64), (2, 32, 1024), (1, 64, 1023), (2, 32, 5), (1, 1, 64 * 1024 + 4096 + 4), (1, 2, 64 * 1024 * 4 + 6)])
def test_wavenet_gate(dev, B, H, T):
    """inputs over +-30 with +-88 and +-200 planted; the float4 path (T % 4 == 0, aligned) and the scalar path (a view
    offset by one float) give the same bits; a row longer than 64 * 1024 wraps the per-row grid-stride loop"""
    g = G.wavenet_gate_inputs(B, H, T, T + H)
    gz = np.random.default_rng(T).standard_normal((B, H, T)).astype(f32)
    z, gg = _gate(dev, g, gz)
    what = f"gate B {B} H {H} T {T}"
    assert np.isfinite(z).all() and np.isfinite(gg).all(), what
    _within("wavenet_gate", what, z, *G.gate(g))
    _within("wavenet_gate_backward", what + " backward", gg, *G.gate_backward(g, gz))
    z1, gg1 = _gate(dev, g, gz, off=1)
    _same(what + " scalar path", z1, z)
    _same(what + " backward scalar path", gg1, gg)
    if T >= 11:  # planted: tanh(0, 88, -88, 200, -200) against sigmoid(-103, 103, -87, 87, -20)
        assert z[0, 0, 1] == 1.0 and z[0, 0, 3] == 1.0 and abs(z[0, 0, 0]) == 0.0 and abs(z[0, 0, 2]) <= 2e-38, (what, z[0, 0, :5])


def test_wavenet_gate_row_limit(dev):
    """65,535 rows is the last supported launch; one more is refused, not run"""
    from parallelwavegan_b200 import capi, ops

    H, T = 65535, 6
    g = G.wavenet_gate_inputs(1, H, T, 3)
    gz = np.random.default_rng(4).standard_normal((1, H, T)).astype(f32)
    z, gg = _gate(dev, g, gz)
    _within("wavenet_gate", "65535 rows", z, *G.gate(g))
    _within("wavenet_gate_backward", "65535 rows backward", gg, *G.gate_backward(g, gz))
    gd = torch.zeros(1, 2 * 65536, 2, device=dev)
    out = torch.zeros(1, 2 * 65536, 2, device=dev)
    L = capi.lib()
    assert L.pwgb_gate_forward(_p(gd), _p(out), 1, 65536, 2, ops._stream()) == -2  # PWGB_UNSUPPORTED
    assert L.pwgb_gate_backward(_p(gd), _p(gd), _p(out), 2, 32768, 2, ops._stream()) == -2
    with pytest.raises(capi.PwgbError, match="too many rows"):
        capi.check(L.pwgb_gate_forward(_p(gd), _p(out), 1, 65536, 2, ops._stream()), "pwgb_gate_forward")


# ---------------------------------------------------------------------------------------------------- loss reductions
@pytest.mark.parametrize("mode", list(G.REDUCE_MODES))
def test_reduce_mean_exact(dev, mode):
    from parallelwavegan_b200 import capi, ops

    L = capi.lib()
    for n in G.REDUCE_SIZES:
        x, y, c, s = G.reduce_data(mode, n, n % 1000 + len(mode))
        xd, yd = _d(x, dev), _d(y, dev) if y is not None else None
        out = ops.reduce_mean_raw(mode, xd, yd, c=c, s=s, weight=0.5)
        _same(f"reduce_mean {mode} n {n}", _n(out)[0], G.reduce_mean_exact(mode, x, y, c, s, 0.5))
        out = _d(np.array([3.0], f32), dev)
        ops.reduce_mean_raw(mode, xd, yd, c=c, s=s, weight=0.25, out=out, accumulate=True)
        _same(f"reduce_mean {mode} n {n} accumulate", _n(out)[0], G.reduce_mean_exact(mode, x, y, c, s, 0.25, prev=3.0))
        xc, yc, _, _ = G.reduce_data(mode, n, n % 1000, coarse=True)
        xcd, ycd = _d(xc, dev), _d(yc, dev) if yc is not None else None
        for ws_floats in (1, 7):  # the grid clamped by the workspace
            ws, out = _nan((ws_floats,), dev), _nan((1,), dev)
            capi.check(L.pwgb_reduce_mean_forward(G.REDUCE_MODES[mode], _p(xcd), _p(ycd), n, c, s, 1.0, 0, _p(out), _p(ws), ws_floats,
                                                  ops._stream()), "pwgb_reduce_mean_forward")
            _same(f"reduce_mean {mode} n {n} ws {ws_floats}", _n(out)[0], G.reduce_mean_exact(mode, xc, yc, c, s, 1.0, ws_floats=ws_floats))
        # backward with weight / n a power of two, overwrite and accumulate
        n2 = 1 << (n - 1).bit_length()
        w = float(f32(n) / f32(n2))  # exact: n < 2^24
        gout = _d(np.array([0.5], f32), dev)
        prev = G.ints(np.random.default_rng(n), n, 4, 1.0 / n2)  # multiples of 2 go, go = 0.5 w / n = 0.5 / n2
        for acc in (0, 1):
            gx = _d(prev, dev) if acc else _nan((n,), dev)
            capi.check(L.pwgb_reduce_mean_backward(G.REDUCE_MODES[mode], _p(xd), _p(yd), n, c, s, w, _p(gout), _p(gx), acc, ops._stream()),
                       "pwgb_reduce_mean_backward")
            _same(f"reduce_mean_backward {mode} n {n} accumulate {acc}", _n(gx),
                  G.reduce_mean_backward_exact(mode, x, y, c, s, w, 0.5, prev if acc else None))


def test_reduce_mean_kinks(dev):
    """hinge inputs exactly on c - s x == 0 and L1 pairs with x == y: term 0, derivative 0"""
    from parallelwavegan_b200 import capi, ops

    x = np.array([1.0, 1.0, 0.5, 1.5, 1.0], f32)
    for mode, y, c, s in (("hinge", None, 1.0, 1.0), ("l1", x.copy(), 0.0, 1.0)):
        xd, yd = _d(x, dev), _d(y, dev) if y is not None else None
        out = _n(ops.reduce_mean_raw(mode, xd, yd, c=c, s=s))[0]
        assert out == (f32(0.1) if mode == "hinge" else f32(0.0))
        gx, gout = _nan((5,), dev), _d(np.array([1.0], f32), dev)
        capi.check(capi.lib().pwgb_reduce_mean_backward(G.REDUCE_MODES[mode], _p(xd), _p(yd), 5, c, s, 5.0, _p(gout), _p(gx), 0, ops._stream()), mode)
        _same(mode + " derivative at the kink", _n(gx), np.array([0, 0, -1, 0, 0], f32) if mode == "hinge" else np.zeros(5, f32))


# ---------------------------------------------------------------------------------------------------- smaller items
@pytest.mark.parametrize("n", [1, 255, 257, 10000])
def test_duration_loss(dev, n):
    from parallelwavegan_b200 import ops

    rng = np.random.default_rng(n)
    x, ds = rng.standard_normal((1, n)).astype(f32), rng.integers(0, 60, (1, n))
    xd, dd = _d(x, dev), _d(ds.astype(np.int64), dev)
    loss, bl, gx, bg = G.duration_loss(x, ds, 1.0)
    _within("duration_loss", f"duration_loss n {n}", _n(ops.duration_loss_raw(xd, dd, 1.0))[0], loss, bl)
    got, gout = _nan((1, n), dev), _d(np.array([1.0], f32), dev)
    _call("pwgb_duration_loss_backward", _p(xd), _p(dd), n, 1.0, _p(gout), _p(got))
    _within("duration_loss", f"duration_loss backward n {n}", _n(got).reshape(-1), gx, bg)


@pytest.mark.parametrize("B,S,K,Cc,one", [(2, 300, 50, 5, True), (3, 257, 8192, 3, False), (1, 1000, 7, 64, False)])
def test_symbol_embed_backward_exact(dev, B, S, K, Cc, one):
    """table gradient bit for bit on exact data: every position on one index (the longest sum), S > 256, and a table at
    the 8192-row limit; one more row is refused"""
    from parallelwavegan_b200 import capi, ops

    rng = np.random.default_rng([B, S, K])
    gy = G.ints(rng, (B, Cc, S), 8, 0.25)
    idx = np.full((B, S), K - 1) if one else rng.integers(0, K, (B, S))
    if not one:
        idx[:, :3] = [0, K - 1, K - 1]
    cd = _d(idx.astype(np.int64).reshape(B, 1, S), dev)
    d_emb, _ = ops.symbol_embed_backward_raw(_d(gy, dev), None, cd, None, S, K)
    _same("symbol_embed_backward", _n(d_emb), G.symbol_embed_backward_exact(gy, idx, K))
    if K == 8192:
        with pytest.raises(capi.PwgbError, match="table rows"):
            ops.symbol_embed_backward_raw(_d(gy, dev), None, cd, None, S, K + 1)
