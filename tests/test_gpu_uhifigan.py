"""UHiFiGAN generator on the GPU: golden parity of forward / inference, the two-source (concat-free) conv-transpose
bit for bit against the single-source entry on torch.cat, the dropout kernel, gradients against oracle autograd,
the f0 / excitation collater, and one reproducible GAN training step of the opencpop recipe."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import REL_TOL, conditioning_tolerances, golden_weights, load_golden, rel_l2
from oracle import ref_ops, synth
from oracle.ref_uhifigan import uhifigan_generator

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _inputs(meta):
    c = synth.randn(tuple(meta["c_shape"]), meta["c_seed"])
    f0 = synth.randn(tuple(meta["f0_shape"]), meta["f0_seed"])
    e = synth.randn(tuple(meta["e_shape"]), meta["e_seed"], meta["e_scale"])
    return c, f0, e


@pytest.mark.parametrize("name", ["uhifigan_small", "uhifigan_opencpop", "uhifigan_odd"])
def test_golden_forward_and_inference(dev, name):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.UHiFiGANGenerator(**meta["kwargs"])
    m.load_state_dict(golden_weights(meta))
    m = m.to(dev).eval()
    c, f0, e = _inputs(meta)
    frames, hop = c.shape[-1], meta["hop"]
    with torch.no_grad():
        y = m(c.to(dev), f0.to(dev), e.to(dev))
        y_inf = m.inference(excitation=e[0].reshape(frames, hop).to(dev), f0=f0[0, 0].to(dev), c=c[0].t().to(dev))
    assert tuple(y.shape) == tuple(g["y"].shape)
    assert rel_l2(y.cpu(), g["y"]) < REL_TOL
    assert tuple(y_inf.shape) == tuple(g["y_inf"].shape)
    assert rel_l2(y_inf.cpu(), g["y_inf"]) < REL_TOL
    m.remove_weight_norm()
    with torch.no_grad():
        assert rel_l2(m(c.to(dev), None, e.to(dev)).cpu(), g["y"]) < REL_TOL


def _plan():
    from parallelwavegan_b200 import capi

    v = (C.c_int * 8)()
    assert capi.lib().pwgb_debug_get(1, v, C.sizeof(v)) == 0
    return dict(zip(("MT", "na", "nb", "ns", "staged", "tma_act", "win_mode", "nco"), list(v)))


# (batch, cin1, cin2, cout, stride, t_in): the four decoder levels of the opencpop recipe, even strides, t_in % 4 != 0,
# a batch of one
CAT_CASES = [
    (2, 512, 512, 256, 3, 40),
    (2, 256, 256, 128, 4, 120),
    (2, 128, 128, 64, 5, 480),
    (2, 64, 64, 32, 5, 2400),
    (2, 64, 64, 32, 2, 300),
    (3, 32, 96, 64, 4, 37),
    (1, 96, 32, 32, 3, 53),
    (1, 256, 256, 128, 2, 64),
]


@pytest.mark.parametrize("variant", [0, 2])  # 2: activations staged by cp.async instead of TMA bulk copies
@pytest.mark.parametrize("B,cin1,cin2,cout,s,T", CAT_CASES)
def test_conv_transpose_cat_bit_identical(dev, B, cin1, cin2, cout, s, T, variant):
    from parallelwavegan_b200 import capi, ops

    K, pad, op = 2 * s, s // 2 + s % 2, s % 2
    x1 = synth.randn((B, cin1, T), 1).to(dev)
    x2 = synth.randn((B, cin2, T), 2).to(dev)
    w = synth.randn((cin1 + cin2, cout, K), 3, 1.0 / math.sqrt(cin1 + cin2)).to(dev)
    b = synth.randn((cout,), 4, 0.1).to(dev)
    t_out = (T - 1) * s - 2 * pad + K + op
    d = capi.ConvTr1dDesc(batch=B, cin=cin1 + cin2, cout=cout, t_in=T, t_out=t_out, kernel=K, stride=s, padding=pad, pre_slope=0.1,
                          groups=1, period=1)
    assert capi.lib().pwgb_conv_transpose1d_cat_supported(C.byref(d), cin1) == 1
    capi.lib().pwgb_debug_set(1, variant)
    try:
        y2 = ops.conv_transpose1d_cat_raw(x1, x2, w, b, stride=s, padding=pad, output_padding=op, pre_slope=0.1)
        plan = _plan()
        y1 = ops.conv_transpose1d_raw(torch.cat((x1, x2), dim=1), w, b, stride=s, padding=pad, output_padding=op, pre_slope=0.1)
    finally:
        capi.lib().pwgb_debug_set(1, 0)
    torch.cuda.synchronize()
    assert plan["ns"] > 0 and plan["tma_act"] == int(variant == 0 and T % 4 == 0)
    assert plan["nco"] >= 1 and (cout * s) % plan["nco"] == 0
    assert tuple(y2.shape) == (B, cout, t_out)
    assert torch.equal(y1, y2)
    ref = F.conv_transpose1d(F.leaky_relu(torch.cat((x1, x2), 1).double(), 0.1), w.double(), b.double(), stride=s, padding=pad,
                             output_padding=op)
    assert rel_l2(y2.cpu(), ref.cpu()) < 1e-5


def test_conv_transpose_cat_empty_batch(dev):
    from parallelwavegan_b200 import ops

    x1 = torch.empty((0, 64, 20), device=dev)
    x2 = torch.empty((0, 64, 20), device=dev)
    w = synth.randn((128, 32, 8), 3).to(dev)
    y = ops.conv_transpose1d_cat_raw(x1, x2, w, None, stride=4, padding=2, pre_slope=0.1)
    assert tuple(y.shape) == (0, 32, 80)
    assert torch.equal(y, ops.conv_transpose1d_raw(torch.cat((x1, x2), 1), w, None, stride=4, padding=2, pre_slope=0.1))


def test_conv_transpose_cat_fallback(dev):
    """x1 with 48 channels (not a multiple of 32): the concatenation is materialised and the single-source entry runs."""
    from parallelwavegan_b200 import capi, ops

    B, cin1, cin2, cout, s, T = 2, 48, 16, 32, 3, 50
    d = capi.ConvTr1dDesc(batch=B, cin=cin1 + cin2, cout=cout, t_in=T, t_out=3 * T, kernel=6, stride=s, padding=2, pre_slope=0.1,
                          groups=1, period=1)
    assert capi.lib().pwgb_conv_transpose1d_cat_supported(C.byref(d), cin1) == 0
    x1, x2 = synth.randn((B, cin1, T), 1), synth.randn((B, cin2, T), 2)
    w, b = synth.randn((cin1 + cin2, cout, 6), 3, 0.2), synth.randn((cout,), 4, 0.1)
    y = ops.conv_transpose1d_cat_raw(x1.to(dev), x2.to(dev), w.to(dev), b.to(dev), stride=s, padding=2, output_padding=1, pre_slope=0.1)
    ref = F.conv_transpose1d(F.leaky_relu(torch.cat((x1, x2), 1), 0.1), w, b, stride=s, padding=2, output_padding=1)
    assert rel_l2(y.cpu(), ref) < 1e-5


def test_dropout_eval_is_identity_without_launches(dev):
    from parallelwavegan_b200 import capi, models, ops

    x = torch.randn(1000, device=dev)
    torch.cuda.synchronize()
    n0 = capi.launch_count()
    assert ops.dropout(x, 0.3, training=False) is x
    assert capi.launch_count() == n0
    meta, _ = load_golden("uhifigan_small")
    sd = golden_weights(meta)
    c, f0, e = (t.to(dev) for t in _inputs(meta))
    outs, counts = [], []
    for p in (0.0, 0.3):
        m = models.UHiFiGANGenerator(**dict(meta["kwargs"], dropout=p))
        m.load_state_dict(sd)
        m = m.to(dev).eval()
        with torch.no_grad():
            m(c, f0, e)  # warm-up: weight packing caches
            capi.reset_launch_count()
            outs.append(m(c, f0, e))
            counts.append(capi.launch_count())
    assert torch.equal(outs[0], outs[1]) and counts[0] == counts[1]


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_training_statistics_and_mask(dev, p):
    from parallelwavegan_b200 import ops

    n = (1 << 22) + 3  # >= 4M elements, with a tail that is not a multiple of 4
    x = (torch.rand(n + 1, device=dev) + 0.5)[1:]  # offset by one element: the unaligned (scalar) path
    scale = torch.tensor(np.float32(1.0) / (np.float32(1.0) - np.float32(p)), device=dev)
    for xx in (x, x.contiguous().clone()):
        y = ops.dropout(xx, p, training=True)
        kept = y != 0
        frac = 1.0 - kept.double().mean().item()
        sigma = math.sqrt(p * (1 - p) / n)
        assert abs(frac - p) < 6 * sigma, (frac, p, sigma)
        assert torch.equal(y[kept], xx[kept] * scale)
    xg = x.clone().requires_grad_(True)
    y = ops.dropout(xg, p, training=True)
    y.backward(torch.ones_like(y))
    assert torch.equal(xg.grad != 0, y != 0)
    assert torch.equal(xg.grad[y != 0], torch.full_like(y, 1.0)[y != 0] * scale)


def test_dropout_seeded_reproducible_and_fresh_per_call(dev):
    from parallelwavegan_b200 import ops

    x = torch.randn(100003, device=dev)
    torch.manual_seed(5)
    a = ops.dropout(x, 0.1, training=True)
    b = ops.dropout(x, 0.1, training=True)
    torch.manual_seed(5)
    a2 = ops.dropout(x, 0.1, training=True)
    with torch.no_grad():  # also applied under no_grad in training mode
        b2 = ops.dropout(x, 0.1, training=True)
    assert torch.equal(a, a2) and torch.equal(b, b2)
    assert not torch.equal(a, b)


def test_uhifigan_gradients(dev):
    """dropout = 0 in train mode: gradients of every parameter and of c / excitation vs torch autograd through the CPU
    oracle, with tolerances from the conditioning of the computation (as the causal HiFi-GAN test)."""
    from parallelwavegan_b200 import models

    kw = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[3, 2], downsample_kernel_sizes=[6, 4],
              upsample_scales=[2, 3], upsample_kernel_sizes=[4, 6], resblock_kernel_sizes=[3, 5], resblock_dilations=[[1, 3], [1, 2]],
              dropout=0.0)
    g = models.UHiFiGANGenerator(**kw)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 19, 1.0)
    g.load_state_dict(sd)
    c = synth.randn((2, 80, 20), 25)
    e = synth.randn((2, 1, 20 * 6), 26, 0.3)
    gout = synth.randn((2, 1, 20 * 6), 27)
    keep = {}

    def oracle(leaves):
        leaf = {k: v.clone().requires_grad_(True) for k, v in leaves.items() if not k.startswith("__")}
        c_ref = leaves["__c"].clone().requires_grad_(True)
        e_ref = leaves["__e"].clone().requires_grad_(True)
        y_ref = uhifigan_generator(ref_ops.fold_weight_norm(leaf), e_ref, c_ref, kw)
        (y_ref * gout).sum().backward()
        keep.setdefault("y", y_ref.detach())
        out = {k: v.grad for k, v in leaf.items()}
        out["__c"], out["__e"] = c_ref.grad, e_ref.grad
        return out

    ref, tol, obs = conditioning_tolerances(oracle, dict(sd, __c=c, __e=e))
    g = g.to(dev).train()
    c_o = c.to(dev).requires_grad_(True)
    e_o = e.to(dev).requires_grad_(True)
    y = g(c_o, None, e_o)
    assert rel_l2(y.detach().cpu(), keep["y"]) < REL_TOL
    (y * gout.to(dev)).sum().backward()
    bad = []
    for k, gr in [("__c", c_o.grad), ("__e", e_o.grad)] + [(k, p.grad) for k, p in g.named_parameters()]:
        err = rel_l2(gr.cpu(), ref[k])
        if err >= tol[k]:
            bad.append((k, round(err, 5), round(tol[k], 5), round(obs[k], 6)))
    assert not bad, bad


HOP = 300


def _corpus_items(n=3, seed=0):
    rng = np.random.RandomState(seed)
    items = []
    for i in range(n):
        frames = 36 + 7 * i
        audio = (0.3 * rng.randn(frames * HOP - (5 if i == 1 else 0))).astype(np.float32)  # item 1: edge-padded by the collater
        items.append((audio, rng.randn(frames, 80).astype(np.float32), rng.rand(frames).astype(np.float32) * 400,
                      (0.1 * rng.randn(frames, HOP)).astype(np.float32)))
    return items


def _reference_collate(items, batch_max_steps, hop, ctx):
    """bin/train.py:725-797 (mel2wav case with f0 / excitation), restated on numpy."""
    frames = batch_max_steps // hop
    start_offset, end_offset, threshold = ctx, -(frames + ctx), frames + 2 * ctx
    batch = []
    for x, c, f, e in items:
        if len(c) <= threshold:
            continue
        if len(x) < len(c) * hop:
            x = np.pad(x, (0, len(c) * hop - len(x)), mode="edge")
        batch.append((x, c, f, e))
    starts = np.array([np.random.randint(start_offset, len(b[1]) + end_offset) for b in batch])
    ys, cs, fs, es = [], [], [], []
    for (x, c, f, e), s in zip(batch, starts):
        ys.append(x[s * hop: s * hop + batch_max_steps])
        cs.append(c[s - ctx: s + frames + ctx])
        fs.append(f[s - ctx: s + frames + ctx])
        es.append(e[s - ctx: s + frames + ctx])
    y = torch.tensor(np.array(ys), dtype=torch.float).unsqueeze(1)
    c = torch.tensor(np.array(cs), dtype=torch.float).transpose(2, 1)
    f = torch.tensor(np.array(fs), dtype=torch.float).unsqueeze(1)
    e = torch.tensor(np.array(es), dtype=torch.float)
    return (c, f, e.reshape(e.shape[0], 1, -1)), y


@pytest.mark.parametrize("ctx", [0, 2])
def test_collater_f0_excitation_matches_reference(dev, ctx):
    from parallelwavegan_b200 import datasets

    items = _corpus_items()
    corpus = datasets.DeviceCorpus(items, dev, hop_size=HOP)
    col = datasets.Collater(batch_max_steps=8400, hop_size=HOP, aux_context_window=ctx, use_f0_and_excitation=True)
    np.random.seed(31)
    (c, f0, e), y = col(corpus, list(range(len(items))))
    np.random.seed(31)
    (c_r, f0_r, e_r), y_r = _reference_collate(items, 8400, HOP, ctx)
    for a, r in ((c, c_r), (f0, f0_r), (e, e_r), (y, y_r)):
        assert tuple(a.shape) == tuple(r.shape)
        assert torch.equal(a.cpu(), r)


OPENCPOP = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[5, 5, 4, 3],
                downsample_kernel_sizes=[10, 10, 8, 6], upsample_scales=[3, 4, 5, 5], upsample_kernel_sizes=[6, 8, 10, 10],
                resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], dropout=0.1,
                use_additional_convs=True, bias=True, nonlinear_activation="LeakyReLU",
                nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)


def _opencpop_step(dev, items):
    """One GanTrainStep of egs/opencpop/voc1/conf/uhifigan.v1.yaml (batch of 2) from fresh seeded weights."""
    from parallelwavegan_b200 import datasets, losses, models, optimizers
    from parallelwavegan_b200.train_step import GanTrainStep

    g = models.UHiFiGANGenerator(**OPENCPOP)
    g.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 41, 1.0))
    d = models.HiFiGANMultiScaleMultiPeriodDiscriminator()
    d.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in d.state_dict().items()], 42, 1.4))
    g, d = g.to(dev).train(), d.to(dev).train()
    crit = {
        "stft": losses.MultiResolutionSTFTLoss(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240]).to(dev),
        "mel": losses.MelSpectrogramLoss(fs=24000, fft_size=2048, hop_size=300, win_length=1200, window="hann", num_mels=80, fmin=0,
                                         fmax=12000, log_base=None).to(dev),
        "gen_adv": losses.GeneratorAdversarialLoss(average_by_discriminators=False),
        "dis_adv": losses.DiscriminatorAdversarialLoss(average_by_discriminators=False),
        "feat_match": losses.FeatureMatchLoss(average_by_layers=False, average_by_discriminators=False, include_final_outputs=False),
    }
    opt_g = optimizers.FusedAdam(g.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    opt_d = optimizers.FusedAdam(d.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    step = GanTrainStep(g, d, crit, opt_g, opt_d, lambda_aux=45.0, lambda_adv=1.0, lambda_feat_match=2.0,
                        generator_train_start_steps=0, discriminator_train_start_steps=0, steps=1)
    corpus = datasets.DeviceCorpus(items, dev, hop_size=HOP)
    col = datasets.Collater(batch_max_steps=8400, hop_size=HOP, aux_context_window=0, use_f0_and_excitation=True)
    np.random.seed(3)
    torch.manual_seed(3)
    x, y = col(corpus, [0, 2])
    stats = step(x, y)
    torch.cuda.synchronize()
    return ({k: float(v) for k, v in stats.items()}, {k: p.grad.clone() for k, p in g.named_parameters()},
            {k: p.detach().clone() for k, p in g.named_parameters()})


def test_opencpop_train_step_reproducible(dev):
    items = _corpus_items()
    s1, g1, p1 = _opencpop_step(dev, items)
    s2, g2, p2 = _opencpop_step(dev, items)
    for k in ("generator_loss", "mel_loss", "spectral_convergence_loss", "log_stft_magnitude_loss", "adversarial_loss",
              "feature_matching_loss", "discriminator_loss", "real_loss", "fake_loss"):
        assert k in s1 and math.isfinite(s1[k]), (k, s1.get(k))
    # the generator phase (every loss computed before the first backward) sees the same batch and the same dropout
    # masks: bit-identical.  The gradients, and the discriminator phase after the update, go through the STFT loss
    # adjoint, whose overlap-add uses float atomics, so they agree to rounding.  Adam's first step moves every weight
    # by about lr in the direction of its gradient's sign, so a gradient within rounding of zero may step either way.
    for k in ("generator_loss", "mel_loss", "spectral_convergence_loss", "log_stft_magnitude_loss", "adversarial_loss",
              "feature_matching_loss"):
        assert s1[k] == s2[k], (k, s1[k], s2[k])
    for k in ("discriminator_loss", "real_loss", "fake_loss"):
        assert abs(s1[k] - s2[k]) <= 1e-5 * abs(s1[k]), (k, s1[k], s2[k])
    for k in p1:
        assert rel_l2(g1[k].cpu(), g2[k].cpu()) < 1e-4, k
        assert float((p1[k] - p2[k]).abs().max()) <= 2 * 2e-4 * (1 + 1e-3), k
