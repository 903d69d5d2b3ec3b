"""Discrete-symbol HiFi-GAN generators on the GPU: golden parity of forward / inference / synthesis, the embed kernel
bit for bit against a CPU gather, LayerNorm / embed backward / duration loss and rounding against torch, gradients
against oracle autograd, the launch count of the front end, the duration collater, and one reproducible cvss_c
training step."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import REL_TOL, conditioning_tolerances, golden_weights, load_golden, rel_l2
from oracle import ref_discrete, ref_ops, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _model(meta, dev):
    from parallelwavegan_b200 import models

    cls = {"dsym_generator": models.DiscreteSymbolHiFiGANGenerator,
           "dsym_duration_generator": models.DiscreteSymbolDurationGenerator}[meta["kind"]]
    m = cls(**meta["kwargs"])
    m.load_state_dict(golden_weights(meta))
    if "linear_bias" in meta:
        with torch.no_grad():
            m.duration_predictor.linear.bias.fill_(meta["linear_bias"])
            m.duration_predictor.linear.weight.mul_(meta["linear_weight_scale"])
    return m.to(dev).eval()


@pytest.mark.parametrize("name", ["dsym_small", "dsym_vctk"])
def test_golden_forward_and_inference(dev, name):
    meta, g = load_golden(name)
    m = _model(meta, dev)
    c = g["c"].to(dev)
    with torch.no_grad():
        y = m(c)
        y_inf = m.inference(c[0].t())
        y_long = m(c.long())  # the duration collater's int64 codes: same indices, same result
    assert tuple(y.shape) == tuple(g["y"].shape) and rel_l2(y.cpu(), g["y"]) < REL_TOL
    assert torch.equal(y, y_long)
    assert rel_l2(y_inf.cpu(), g["y_inf"]) < REL_TOL
    if "y_inf_g" in g:
        with torch.no_grad():
            assert rel_l2(m.inference(c[0].t().cpu().numpy(), g=meta["g"]).cpu(), g["y_inf_g"]) < REL_TOL
    m.remove_weight_norm()
    with torch.no_grad():
        assert rel_l2(m(c).cpu(), g["y"]) < REL_TOL


@pytest.mark.parametrize("name", ["dsym_dur_cvss", "dsym_dur_odd"])
def test_golden_duration_generator(dev, name):
    meta, g = load_golden(name)
    m = _model(meta, dev)
    c, ds = g["c"].to(dev), g["ds"].to(dev)
    with torch.no_grad():
        y, ds_out = m(c, ds.clone())
        y_syn, ds_syn = m.synthesis(c)
        y_inf = m.inference(c[0].t())
        y_inf_ds = m.inference(c[0].t(), ds=ds[0].clone())
    assert tuple(y.shape) == tuple(g["y"].shape) and rel_l2(y.cpu(), g["y"]) < REL_TOL
    assert rel_l2(ds_out.cpu(), g["ds_out"]) < REL_TOL
    assert ds_syn.dtype == torch.int64 and torch.equal(ds_syn.cpu(), g["ds_syn"])
    assert tuple(y_syn.shape) == tuple(g["y_syn"].shape) and rel_l2(y_syn.cpu(), g["y_syn"]) < REL_TOL
    assert tuple(y_inf.shape) == tuple(g["y_inf"].shape) and rel_l2(y_inf.cpu(), g["y_inf"]) < REL_TOL
    assert tuple(y_inf_ds.shape) == tuple(g["y_inf_ds"].shape) and rel_l2(y_inf_ds.cpu(), g["y_inf_ds"]) < REL_TOL


def _cpu_embed(c, table, spk=None, ds=None):
    """torch gather (+ speaker add), then repeat_interleave and zero padding: the reference's front end on the CPU."""
    ci = c.long()
    e = F.embedding(ci[:, 0], table).transpose(1, 2)
    if spk is not None:
        e = e + F.embedding(ci[:, 1, 0], spk)[:, :, None]
    if ds is None:
        return e
    rows = [torch.repeat_interleave(x, d, dim=1) for x, d in zip(e, ds)]
    out = e.new_zeros(e.shape[0], e.shape[1], max([r.shape[1] for r in rows] + [0]))
    for b, r in enumerate(rows):
        out[b, :, : r.shape[1]] = r
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.int64])
@pytest.mark.parametrize("spk", [False, True])
@pytest.mark.parametrize("durations", [False, True])
def test_embed_bit_identical_to_gather(dev, dtype, spk, durations):
    from parallelwavegan_b200 import ops

    B, S, C, E, G = 3, 45, 200, 37, 5
    rng = np.random.RandomState(3)
    c = torch.from_numpy(rng.randint(0, E, size=(B, 2 if spk else 1, S))).to(dtype)
    if spk:
        c[:, 1] = torch.from_numpy(rng.randint(0, G, size=(B, 1)))
    if dtype == torch.float32:
        c[:, 0] += 0.7  # c.long() truncates
    table = synth.randn((E, C), 1)
    spk_t = synth.randn((G, C), 2) if spk else None
    ds = None
    if durations:  # zero-duration symbols and ragged row totals
        ds = torch.from_numpy(rng.randint(0, 4, size=(B, S))).long()
        ds[1, 10:] = 0
        ds[2, :5] = 0
    ref = _cpu_embed(c, table, spk_t, ds)
    dsd = ds.to(dev) if ds is not None else None
    y = ops.symbol_embed_raw(c.to(dev), table.to(dev), spk_t.to(dev) if spk else None, ds=dsd,
                             t_out=int(ds.sum(1).max()) if durations else None)
    assert tuple(y.shape) == tuple(ref.shape)
    assert torch.equal(y.cpu(), ref)


def test_embed_strided_index_empty_batch_and_out_of_range(dev):
    from parallelwavegan_b200 import capi, ops

    table, spk_t = synth.randn((10, 64), 1).to(dev), synth.randn((3, 64), 2).to(dev)
    c = torch.tensor([[1, 2], [4, 2], [9, 2]], device=dev)  # (T, 2) as inference builds it: a (1, 2, T) view of stride 2
    y = ops.symbol_embed_raw(c.t().unsqueeze(0), table, spk_t)
    assert torch.equal(y.cpu(), _cpu_embed(c.t().unsqueeze(0).cpu(), table.cpu(), spk_t.cpu()))
    torch.cuda.synchronize()
    n0 = capi.launch_count()
    y = ops.symbol_embed_raw(torch.empty((0, 1, 7), device=dev), table)
    assert tuple(y.shape) == (0, 64, 7) and capi.launch_count() == n0
    # an index outside the table is never read: its column is NaN, the others are exact
    c = torch.tensor([[[3, 10, -1, 0, 9]]], device=dev)
    y = ops.symbol_embed_raw(c, table).cpu()
    assert torch.isnan(y[0, :, 1]).all() and torch.isnan(y[0, :, 2]).all()
    ok = [0, 3, 4]
    assert torch.equal(y[0][:, ok], table.cpu()[[3, 0, 9]].t())
    # a speaker outside its table: the whole item is NaN
    c = torch.tensor([[[1, 2], [5, 5]], [[1, 2], [0, 0]]], device=dev)
    y = ops.symbol_embed_raw(c, table, spk_t).cpu()
    assert torch.isnan(y[0]).all() and not torch.isnan(y[1]).any()


def test_channel_layernorm_forward_backward(dev):
    from parallelwavegan_b200 import ops

    for B, C, T in ((3, 384, 45), (2, 64, 1), (1, 100, 70)):
        x = synth.randn((B, C, T), 5) * 3 + 0.5
        gm, bt = synth.randn((C,), 6), synth.randn((C,), 7, 0.1)
        gy = synth.randn((B, C, T), 8)
        xd = x.double().requires_grad_(True)
        gmd, btd = gm.double().requires_grad_(True), bt.double().requires_grad_(True)
        ref = F.layer_norm(xd.transpose(1, 2), (C,), gmd, btd, 1e-12).transpose(1, 2)
        (ref * gy.double()).sum().backward()
        xg = x.to(dev).requires_grad_(True)
        g2, b2 = gm.to(dev).requires_grad_(True), bt.to(dev).requires_grad_(True)
        y = ops.channel_layer_norm(xg, g2, b2, 1e-12)
        (y * gy.to(dev)).sum().backward()
        assert rel_l2(y.detach().cpu(), ref.detach()) < 1e-5
        for a, r in ((xg.grad, xd.grad), (g2.grad, gmd.grad), (b2.grad, btd.grad)):
            assert rel_l2(a.cpu(), r) < 1e-5


@pytest.mark.parametrize("durations", [False, True])
def test_embed_backward_against_autograd_and_deterministic(dev, durations):
    from parallelwavegan_b200 import ops

    B, S, C, E, G = 4, 60, 96, 13, 3
    rng = np.random.RandomState(11)
    c = torch.from_numpy(rng.randint(0, E, size=(B, 2, S)))
    c[:, 1] = torch.from_numpy(rng.randint(0, G, size=(B, 1)))
    ds = torch.from_numpy(rng.randint(0, 4, size=(B, S))).long() if durations else None
    table, spk_t = synth.randn((E, C), 1), synth.randn((G, C), 2)
    t_out = int(ds.sum(1).max()) if durations else S
    gy, gsym = synth.randn((B, C, t_out), 3), synth.randn((B, C, S), 4)
    td, sd = table.double().requires_grad_(True), spk_t.double().requires_grad_(True)
    e = _cpu_embed(c, td, sd)
    loss = (_cpu_embed(c, td, sd, ds) * gy.double()).sum() + ((e * gsym.double()).sum() if durations else 0)
    loss.backward()
    grads = []
    for _ in range(2):
        tg, sg = table.to(dev).requires_grad_(True), spk_t.to(dev).requires_grad_(True)
        out = ops.symbol_embed(c.to(dev), tg, sg, ds=ds.to(dev) if durations else None, t_out=t_out, symbol_level=durations)
        if durations:
            y, y_sym = out
            ((y * gy.to(dev)).sum() + (y_sym * gsym.to(dev)).sum()).backward()
        else:
            (out * gy.to(dev)).sum().backward()
        grads.append((tg.grad.clone(), sg.grad.clone()))
    assert rel_l2(grads[0][0].cpu(), td.grad) < 1e-5 and rel_l2(grads[0][1].cpu(), sd.grad) < 1e-5
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    unused = sorted(set(range(E)) - set(c[:, 0].unique().tolist()))
    assert all(not grads[0][0][u].any() for u in unused)


def test_duration_loss_and_rounding(dev):
    from parallelwavegan_b200 import losses, ops

    x = synth.randn((3, 17), 9)
    ds = torch.from_numpy(np.random.RandomState(1).randint(0, 6, size=(3, 17))).long()
    xd = x.to(dev).requires_grad_(True)
    loss = losses.DurationPredictorLoss(offset=1.0)(xd, ds.to(dev))
    loss.backward()
    xr = x.double().requires_grad_(True)
    ref = F.mse_loss(xr, torch.log(ds.double() + 1.0))
    ref.backward()
    assert loss.dim() == 0 and abs(float(loss) - float(ref)) <= 1e-6 * float(ref)
    assert rel_l2(xd.grad.cpu(), xr.grad) < 1e-5
    # rounding: torch.round is half to even; keep away from the boundaries fp32 exp may straddle
    v = torch.tensor([[0.2, 1.0, 1.5, 2.5, 3.4999, 0.0, 7.9], [0.49, 0.51, 2.0, 4.5, 1.01, 0.3, 5.5]])
    xv = torch.log(v + 1.0)
    d, tot = ops.duration_round(xv.to(dev), 1.0)
    ref_d = ref_discrete.duration_round(xv, 1.0)
    assert torch.equal(d.cpu(), ref_d) and torch.equal(tot.cpu(), ref_d.sum(1))


def test_duration_zero_rule_matches_oracle(dev):
    from parallelwavegan_b200 import ops

    x = torch.full((3, 5), -3.0)  # every duration rounds to 0
    d, tot = ops.duration_round(x.to(dev), 1.0)
    e = torch.randn(3, 4, 5)
    ref_ds = ref_discrete.duration_round(x, 1.0)
    ref_discrete.length_regulate(e, ref_ds)
    assert torch.equal(d.cpu(), ref_ds) and torch.equal(tot.cpu(), torch.full((3,), 5))
    ds = torch.tensor([[0, 0, 0], [1, 0, 2]], device=dev)  # the batch does not sum to zero: nothing changes
    _, tot = ops.duration_round(None, ds=ds)
    assert torch.equal(ds.cpu(), torch.tensor([[0, 0, 0], [1, 0, 2]])) and tot.tolist() == [0, 3]
    d, _ = ops.duration_round(x.to(dev), 1.0, zero_rule=False)
    assert not d.any()


def _grad_check(dev, m, oracle_fn, inputs, sd, extra=()):
    keep = {}

    def oracle(leaves):
        leaf = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
        outs = oracle_fn(ref_ops.fold_weight_norm(leaf), *inputs)
        loss = sum((o * go).sum() for o, go in zip(outs, extra))
        loss.backward()
        keep.setdefault("outs", [o.detach() for o in outs])
        return {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaf.items()}

    ref, tol, obs = conditioning_tolerances(oracle, dict(sd))
    return ref, tol, obs, keep


def test_dsym_generator_gradients(dev):
    from parallelwavegan_b200 import models

    kw = dict(in_channels=64, channels=64, num_embs=12, num_spk_embs=4, spk_emb_dim=64, kernel_size=7, upsample_scales=[4, 2],
              upsample_kernel_sizes=[8, 4], resblock_kernel_sizes=[3, 5], resblock_dilations=[[1, 3], [1, 2]])
    g = models.DiscreteSymbolHiFiGANGenerator(**kw)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 23, 1.0)
    g.load_state_dict(sd)
    rng = np.random.RandomState(5)
    c = torch.from_numpy(rng.randint(0, 12, size=(2, 2, 16))).float()
    c[:, 1] = torch.tensor([[1.0], [3.0]])
    gout = synth.randn((2, 1, 16 * 8), 27)
    ref, tol, obs, keep = _grad_check(dev, g, lambda w, cc: [ref_discrete.dsym_generator(w, cc, kw)], [c], sd, [gout])
    g = g.to(dev).train()
    y = g(c.to(dev))
    assert rel_l2(y.detach().cpu(), keep["outs"][0]) < REL_TOL
    (y * gout.to(dev)).sum().backward()
    bad = [(k, rel_l2(p.grad.cpu(), ref[k]), tol[k]) for k, p in g.named_parameters() if rel_l2(p.grad.cpu(), ref[k]) >= tol[k]]
    assert not bad, bad


def test_dsym_duration_generator_gradients(dev):
    from parallelwavegan_b200 import models

    kw = dict(in_channels=64, channels=64, num_embs=12, num_spk_embs=0, kernel_size=7, upsample_scales=[4, 2], upsample_kernel_sizes=[8, 4],
              resblock_kernel_sizes=[3, 5], resblock_dilations=[[1, 3], [1, 2]], duration_chans=96, duration_dropout_rate=0.0)
    g = models.DiscreteSymbolDurationGenerator(**kw)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 29, 1.0)
    g.load_state_dict(sd)
    rng = np.random.RandomState(8)
    c = torch.from_numpy(rng.randint(0, 13, size=(2, 1, 14)))
    ds = torch.from_numpy(rng.randint(0, 4, size=(2, 14))).long()  # zero durations, ragged totals 27 / 22
    t_out = int(ds.sum(1).max())
    assert t_out % 16 and bool(ds.eq(0).any()) and len(set(ds.sum(1).tolist())) == 2
    gout, gds = synth.randn((2, 1, t_out * 8), 31), synth.randn((2, 14), 32)
    # Every frame of input_conv's output reaches the first LeakyReLU, and the input_conv / embedding gradients sum over
    # all of them, so a single pre-activation within rounding of 0 flips the derivative (1 vs 0.1) of one element and
    # moves those gradients by percents: with RandomState(6) one element is 9.3e-7, the tensor-core forward lands on the
    # other side of 0 and input_conv.bias moves by 4.3 %, the full size of that element's flipped term.  Such data
    # measures the kink, not the kernels; keep the pre-activations clear of it (the forward agrees to ~1e-6 here).
    w0 = ref_ops.fold_weight_norm(sd)
    h0 = F.conv1d(ref_discrete.length_regulate(ref_discrete.embed(w0, c, kw), ds.clone()), w0["input_conv.weight"],
                  w0["input_conv.bias"], padding=3)
    assert float(h0.abs().min()) > 1e-4

    def fn(w, cc):
        y, d = ref_discrete.dsym_duration_forward(w, cc, ds.clone(), kw)
        return [y, d]

    ref, tol, obs, keep = _grad_check(dev, g, fn, [c], sd, [gout, gds])
    g = g.to(dev).train()
    y, d = g(c.to(dev), ds.to(dev))
    assert rel_l2(y.detach().cpu(), keep["outs"][0]) < REL_TOL and rel_l2(d.detach().cpu(), keep["outs"][1]) < REL_TOL
    ((y * gout.to(dev)).sum() + (d * gds.to(dev)).sum()).backward()
    bad = [(k, rel_l2(p.grad.cpu(), ref[k]), tol[k]) for k, p in g.named_parameters() if rel_l2(p.grad.cpu(), ref[k]) >= tol[k]]
    assert not bad, bad


@pytest.mark.parametrize("T", [16, 24, 27])
def test_first_upsample_backward_at_regulated_lengths(dev, T):
    """The conv-transpose after input_conv (64 -> 32, k 8, stride 4, LeakyReLU 0.1 fused) at the regulated lengths of the
    duration tests: data, weight and bias gradients against float64 torch."""
    from parallelwavegan_b200 import ops

    x, w, b = synth.randn((2, 64, T), 1, 0.3), synth.randn((64, 32, 8), 2, 0.1), synth.randn((32,), 3, 0.1)
    gy = synth.randn((2, 32, 4 * T), 4)
    xd, wd, bd = (t.to(dev).requires_grad_(True) for t in (x, w, b))
    ops.conv_transpose1d(xd, wd, bd, stride=4, padding=2, pre_slope=0.1).backward(gy.to(dev))
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    F.conv_transpose1d(F.leaky_relu(xr, 0.1), wr, br, stride=4, padding=2).backward(gy.double())
    for a, r in ((xd, xr), (wd, wr), (bd, br)):
        assert rel_l2(a.grad.cpu(), r.grad) < 2e-5


def test_length_regulator_module(dev):
    from parallelwavegan_b200 import layers

    xs = synth.randn((2, 5, 8), 1).to(dev)
    ds = torch.tensor([[1, 0, 2, 1, 0], [3, 1, 0, 0, 1]], device=dev)
    y = layers.LengthRegulator()(xs, ds)
    ref = _cpu_embed(torch.arange(10).reshape(2, 1, 5), xs.cpu().reshape(10, 8), ds=ds.cpu()).transpose(1, 2)
    assert tuple(y.shape) == (2, 5, 8) and torch.equal(y.cpu(), ref)
    assert tuple(layers.LengthRegulator()(xs[:0], ds[:0]).shape) == (0, 0, 8)


def test_front_end_is_one_launch(dev):
    """An eval forward of DiscreteSymbolHiFiGANGenerator is the HiFiGANGenerator body on the embedding plus one launch."""
    from parallelwavegan_b200 import capi, models, ops

    meta, g = load_golden("dsym_vctk")
    m = _model(meta, dev)
    kw = {k: v for k, v in meta["kwargs"].items() if k not in ("num_embs", "num_spk_embs", "spk_emb_dim", "concat_spk_emb")}
    h = models.HiFiGANGenerator(**kw)
    h.load_state_dict({k: v for k, v in m.state_dict().items() if not k.startswith(("emb.", "spk_emb."))})
    h = h.to(dev).eval()
    c = g["c"].to(dev)
    counts = []
    with torch.no_grad():
        e = ops.symbol_embed_raw(c, m.emb.weight, m.spk_emb.weight)
        for f, x in ((m, c), (h, e)):
            f(x)  # warm-up: weight packing caches
            torch.cuda.synchronize()
            capi.reset_launch_count()
            out = f(x)
            torch.cuda.synchronize()
            counts.append((capi.launch_count(), out))
    assert counts[0][0] == counts[1][0] + 1, counts
    assert torch.equal(counts[0][1], counts[1][1])


HOP = 320


def _dur_items(n=3, seed=0, channels=1, num_embs=50):
    rng = np.random.RandomState(seed)
    items = []
    for i in range(n):
        frames = 40 + 9 * i
        codes = np.repeat(rng.randint(0, num_embs, size=(frames, channels)), rng.randint(1, 4, size=frames), axis=0)[:frames]
        items.append(((0.3 * rng.randn(frames * HOP)).astype(np.float32), codes.astype(np.float32) + 0.25))
    return items


def _reference_duration_collate(items, batch_max_steps, hop, ctx, pad_value):
    """bin/train.py:725-783 (mel2wav case with durations), restated on numpy / torch."""
    frames = batch_max_steps // hop
    start_offset, end_offset, threshold = ctx, -(frames + ctx), frames + 2 * ctx
    batch = [(x, c) for x, c in items if len(c) > threshold]
    starts = np.array([np.random.randint(start_offset, len(c) + end_offset) for _, c in batch])
    ys, codes, lens = [], [], []
    for (x, c), s in zip(batch, starts):
        ys.append(x[s * hop: s * hop + batch_max_steps])
        code, d = torch.unique_consecutive(torch.tensor(c[s - ctx: s + frames + ctx], dtype=torch.long), return_counts=True, dim=0)
        codes.append(code)
        lens.append(d)
    S = max(len(d) for d in lens)
    cb = torch.full((len(codes), S, codes[0].shape[1]), pad_value, dtype=torch.long)
    db = torch.zeros((len(lens), S), dtype=torch.long)
    for i, (cc, d) in enumerate(zip(codes, lens)):
        cb[i, : len(cc)] = cc
        db[i, : len(d)] = d
    return cb.transpose(2, 1), torch.tensor(np.array(ys), dtype=torch.float).unsqueeze(1), db


@pytest.mark.parametrize("channels,ctx", [(1, 0), (2, 2)])
def test_duration_collater_matches_reference(dev, channels, ctx):
    from parallelwavegan_b200 import datasets

    items = _dur_items(channels=channels)
    corpus = datasets.DeviceCorpus(items, dev, hop_size=HOP)
    col = datasets.Collater(batch_max_steps=10240, hop_size=HOP, aux_context_window=ctx, use_duration=True, pad_value=50)
    np.random.seed(17)
    c, y, ds = col(corpus, list(range(len(items))))
    np.random.seed(17)
    c_r, y_r, ds_r = _reference_duration_collate(items, 10240, HOP, ctx, 50)
    for a, r in ((c, c_r), (y, y_r), (ds, ds_r)):
        assert a.dtype == r.dtype and tuple(a.shape) == tuple(r.shape)
        assert torch.equal(a.cpu(), r)


CVSS = dict(in_channels=512, out_channels=1, channels=512, num_embs=500, kernel_size=7, upsample_scales=[10, 8, 2, 2],
            upsample_kernel_sizes=[20, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
            use_additional_convs=True, bias=True, nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
            use_weight_norm=True, duration_layers=2, duration_chans=384, duration_kernel_size=3, duration_offset=1.0,
            duration_dropout_rate=0.5, num_spk_embs=0)


def _cvss_step(dev, items):
    """One GanTrainStep of egs/cvss_c/hubert_voc1/conf/hifigan_hubert_duration.v1.yaml (batch of 2) from seeded weights."""
    from parallelwavegan_b200 import datasets, losses, models, optimizers
    from parallelwavegan_b200.train_step import GanTrainStep

    g = models.DiscreteSymbolDurationGenerator(**CVSS)
    g.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 51, 1.0))
    d = models.HiFiGANMultiScaleMultiPeriodDiscriminator()
    d.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in d.state_dict().items()], 52, 1.4))
    g, d = g.to(dev).train(), d.to(dev).train()
    crit = {
        "duration": losses.DurationPredictorLoss(offset=1.0),
        "mel": losses.MelSpectrogramLoss(fs=16000, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80, fmin=0,
                                         fmax=8000, log_base=None).to(dev),
        "gen_adv": losses.GeneratorAdversarialLoss(average_by_discriminators=False),
        "dis_adv": losses.DiscriminatorAdversarialLoss(average_by_discriminators=False),
        "feat_match": losses.FeatureMatchLoss(average_by_layers=False, average_by_discriminators=False, include_final_outputs=False),
    }
    opt_g = optimizers.FusedAdam(g.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    opt_d = optimizers.FusedAdam(d.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    step = GanTrainStep(g, d, crit, opt_g, opt_d, lambda_aux=45.0, lambda_adv=1.0, lambda_feat_match=2.0,
                        generator_train_start_steps=0, discriminator_train_start_steps=0, steps=1)
    corpus = datasets.DeviceCorpus(items, dev, hop_size=HOP)
    col = datasets.Collater(batch_max_steps=10240, hop_size=HOP, aux_context_window=0, use_duration=True, pad_value=CVSS["num_embs"])
    np.random.seed(3)
    torch.manual_seed(3)
    x, y, ds = col(corpus, [0, 2])
    stats = step(x, y, ds)
    torch.cuda.synchronize()
    return {k: float(v) for k, v in stats.items()}, {k: p.grad.clone() for k, p in g.named_parameters() if p.grad is not None}


def test_cvss_train_step_reproducible(dev):
    items = _dur_items(num_embs=500)
    s1, g1 = _cvss_step(dev, items)
    s2, g2 = _cvss_step(dev, items)
    for k in ("generator_loss", "duration_loss", "mel_loss", "adversarial_loss", "feature_matching_loss", "discriminator_loss",
              "real_loss", "fake_loss"):
        assert k in s1 and math.isfinite(s1[k]), (k, s1.get(k))
    # the generator phase (every loss computed before the first backward) is bit-identical; the rest goes through the
    # STFT adjoint's float atomics (see the opencpop step test)
    for k in ("generator_loss", "duration_loss", "mel_loss", "adversarial_loss", "feature_matching_loss"):
        assert s1[k] == s2[k], (k, s1[k], s2[k])
    for k in ("discriminator_loss", "real_loss", "fake_loss"):
        assert abs(s1[k] - s2[k]) <= 1e-5 * abs(s1[k]), (k, s1[k], s2[k])
    assert "emb.weight" in g1 and "duration_predictor.linear.weight" in g1
    for k in g1:
        assert rel_l2(g1[k].cpu(), g2[k].cpu()) < 1e-4, k
