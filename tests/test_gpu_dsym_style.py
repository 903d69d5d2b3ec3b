"""Discrete-symbol StyleMelGAN generator on the GPU: forward and inference against the real-reference goldens and the
oracle, the speaker argument, weight-norm removal, the launches of the front end and of the whole forward, gradients
against float64 oracle autograd, a reproducible train step on unit batches, and the decoder against ``inference``.

Tolerances are those of ``test_gpu_stylemelgan.py``: the instance-normalised, gated stack is ill-conditioned, so a model
deeper than 4 blocks is held to REL_TOL rel-L2 and 2e-2 of peak pointwise, the others to REL_TOL on both."""
import json
import math

import numpy as np
import pytest
import torch

from helpers import REL_TOL, conditioning_tolerances, golden_weights, load_golden, max_abs_over_peak, rel_l2
from oracle import ref_dsym_style, synth

pytestmark = pytest.mark.gpu
NAMES = ["dsym_style_small", "dsym_style_vctk"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _model(meta, dev):
    from parallelwavegan_b200 import models

    m = models.DiscreteSymbolStyleMelGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    return m.to(dev).eval()


def _close(y, ref, deep):
    return rel_l2(y, ref) < REL_TOL and max_abs_over_peak(y, ref) < (2e-2 if deep else REL_TOL)


def _fold64(sd):
    """w = g * v / ||v|| (torch.nn.utils.weight_norm, dim 0) in the leaves' dtype, so float64 autograd stays float64"""
    out = {k: v for k, v in sd.items() if not k.endswith(("_g", "_v"))}
    out.update({k[: -len("_g")]: torch._weight_norm(sd[k[: -len("_g")] + "_v"], v, 0) for k, v in sd.items() if k.endswith("_g")})
    return out


def _w64(meta):
    return _fold64({k: v.double() for k, v in golden_weights(meta).items()})


@pytest.mark.parametrize("name", NAMES)
def test_forward_matches_reference(dev, name):
    meta, g = load_golden(name)
    m = _model(meta, dev)
    deep = len(meta["kwargs"]["upsample_scales"]) > 4
    c, z = g["c"].to(dev), g["z"].to(dev)
    n = g["x1"].shape[-1]
    with torch.no_grad():
        x0 = m._noise_path(z)
        x1, c1 = m.blocks[0](x0, m._embed(c))
        y = m(c, z)
        y_long = m(c.long(), z)  # int64 codes: the same indices, the same result
    assert rel_l2(x0.cpu(), g["x0"]) < REL_TOL
    assert rel_l2(x1[..., :n].cpu(), g["x1"]) < REL_TOL and rel_l2(c1[..., :n].cpu(), g["c1"]) < REL_TOL
    assert tuple(y.shape) == tuple(g["y"].shape) and _close(y.cpu(), g["y"], deep)
    assert torch.equal(y, y_long)
    ref = ref_dsym_style.dsym_style_generator(_w64(meta), g["c"], g["z"].double(), meta["kwargs"])
    assert _close(y.cpu(), ref, deep)
    m.remove_weight_norm()
    with torch.no_grad():
        assert _close(m(c, z).cpu(), g["y"], deep)


@pytest.mark.parametrize("name", NAMES)
def test_inference_matches_reference(dev, name):
    """inference crops the upsampled noise to T frames: at T a multiple of the noise factor and at one that is not."""
    meta, g = load_golden(name)
    m = _model(meta, dev)
    deep = len(meta["kwargs"]["upsample_scales"]) > 4
    hop = int(np.prod(meta["kwargs"]["upsample_scales"]))
    w = _w64(meta)
    for k, T in enumerate(meta["inf_lengths"]):
        c, noise = g[f"inf{k}_c"], g[f"inf{k}_noise"]
        with torch.no_grad():
            y = m.inference(c.to(dev), noise=noise.to(dev))
        assert tuple(y.shape) == (T * hop, 1)
        assert _close(y.cpu(), g[f"inf{k}_y"], deep), (k, rel_l2(y.cpu(), g[f"inf{k}_y"]))
        assert _close(y.cpu(), ref_dsym_style.dsym_style_inference(w, c, noise.double(), meta["kwargs"]), deep)
        if f"inf{k}_y_g" in g:
            cg = c.clone()
            cg[:, 1] = meta["g"]
            with torch.no_grad():
                y_g = m.inference(c[:, :1].numpy(), g=meta["g"], noise=noise.to(dev))
                assert torch.equal(y_g, m.inference(cg.to(dev), noise=noise.to(dev)))
            assert _close(y_g.cpu(), g[f"inf{k}_y_g"], deep)


def _profile_kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset"))]
    return out, names


def test_front_end_is_one_launch_and_forward_is_libpwgb_only(dev):
    """An eval forward is StyleMelGANGenerator's on the embedding plus one embed launch, and every kernel it runs (weight
    norm removed, so no weight preprocessing) is a libpwgb launch."""
    from parallelwavegan_b200 import capi, models, ops

    meta, g = load_golden("dsym_style_vctk")
    m = _model(meta, dev)
    m.remove_weight_norm()
    kw = {k: v for k, v in meta["kwargs"].items() if k not in ("num_embs", "num_spk_embs", "spk_emb_dim", "concat_spk_emb")}
    s = models.StyleMelGANGenerator(**dict(json.loads(json.dumps(kw)), use_weight_norm=False))
    s.load_state_dict({k: v for k, v in m.state_dict().items() if not k.startswith(("emb.", "spk_emb."))}, strict=True)
    s = s.to(dev).eval()
    c, z = g["c"].to(dev), g["z"].to(dev)
    counts = []
    with torch.no_grad():
        e = ops.symbol_embed_raw(c, m.emb.weight, m.spk_emb.weight)
        for f, x in ((m, c), (s, e)):
            f(x, z)  # warm-up: weight packing caches
            torch.cuda.synchronize()
            capi.reset_launch_count()
            out = f(x, z)
            torch.cuda.synchronize()
            counts.append((capi.launch_count(), out))
        assert counts[0][0] == counts[1][0] + 1, counts
        assert torch.equal(counts[0][1], counts[1][1])
        capi.reset_launch_count()
        _, names = _profile_kernels(lambda: m(c, z))
        n = capi.launch_count()
    assert len(names) == n == counts[0][0], (len(names), n, sorted(set(names)))
    assert not [k for k in names if "at::" in k or "native" in k], sorted(set(names))


def test_gradients_match_oracle_autograd(dev):
    """Every parameter's gradient, the two embedding tables' included (pwgb_symbol_embed_backward), against float64 autograd
    through the oracle, with the conditioning-aware bound of the StyleMelGAN gradient test."""
    from parallelwavegan_b200 import models

    meta, g = load_golden("dsym_style_small")
    kw = json.loads(json.dumps(meta["kwargs"]))
    m = models.DiscreteSymbolStyleMelGANGenerator(**kw)
    sd = golden_weights(meta)
    m.load_state_dict(sd, strict=True)
    c, z = g["c"], g["z"]
    keep = {}

    def oracle(leaves):
        lf = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
        y = ref_dsym_style.dsym_style_generator(_fold64(lf), c, z.double(), kw)
        keep.setdefault("y", y.detach())
        keep.setdefault("t", synth.randn(tuple(y.shape), 77).double())
        (y * keep["t"]).sum().backward()
        return {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in lf.items()}

    ref, tol, obs = conditioning_tolerances(oracle, {k: v.double() for k, v in sd.items()}, rel_eps=2e-5)
    m = m.to(dev).train()
    y = m(c.to(dev), z.to(dev))
    assert rel_l2(y.detach().cpu(), keep["y"]) < REL_TOL
    (y * keep["t"].float().to(dev)).sum().backward()
    grads = {k: p.grad for k, p in m.named_parameters()}
    assert grads["emb.weight"] is not None and grads["spk_emb.weight"] is not None
    assert sorted(grads) == sorted(ref)
    bad = [(k, round(rel_l2(gr.cpu(), ref[k]), 5), round(tol[k], 5), round(obs[k], 6)) for k, gr in grads.items()
           if rel_l2(gr.cpu(), ref[k]) >= tol[k]]
    assert not bad, bad[:10]
    # the speaker table gets only the rows of the batch's speakers, the symbol table only the rows of its symbols
    used = set(c[:, 1, 0].long().tolist())
    assert all(bool(grads["spk_emb.weight"][r].any()) == (r in used) for r in range(kw["num_spk_embs"]))
    unused = sorted(set(range(kw["num_embs"])) - set(c[:, 0].long().unique().tolist()))
    assert all(not grads["emb.weight"][u].any() for u in unused)


# the recipe's generator at a quarter of its width, with its noise and upsampling scales (hop 320, 56 frames per
# noise frame) and the recipe's discriminator and losses
SMALL_RECIPE = dict(in_channels=32, aux_channels=32, channels=32, out_channels=1, num_embs=20, num_spk_embs=4, spk_emb_dim=32,
                    kernel_size=9, dilation=2, noise_upsample_scales=[7, 2, 2, 2], upsample_scales=[5, 2, 2, 2, 2, 2, 2, 1, 1],
                    gated_function="softmax")
HOP = 320
LR_G = 1e-4


def _items(n=3, seed=0):
    rng = np.random.RandomState(seed)
    items = []
    for i in range(n):
        frames = 70 + 11 * i
        codes = np.repeat(rng.randint(0, 20, size=frames), rng.randint(1, 4, size=frames))[:frames]
        units = np.stack([codes, np.full(frames, i % 4)], axis=1).astype(np.float32)
        items.append(((0.3 * rng.randn(frames * HOP)).astype(np.float32), units))
    return items


def _train_step(dev, items):
    """One GanTrainStep of egs/vctk/hubert_voc1/conf/style_melgan_hubert.v1.yaml's loss wiring (MR-STFT + mse adversarial,
    not averaged by discriminators, Adam) on a unit batch from the device collater."""
    from parallelwavegan_b200 import datasets, losses, models, optimizers
    from parallelwavegan_b200.train_step import GanTrainStep

    g = models.DiscreteSymbolStyleMelGANGenerator(**SMALL_RECIPE)
    g.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 71, 1.0))
    d = models.StyleMelGANDiscriminator(repeats=4)
    d.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in d.state_dict().items() if not k.endswith("_filter")], 72, 1.4),
                      strict=False)
    g, d = g.to(dev).train(), d.to(dev).train()
    crit = {
        "stft": losses.MultiResolutionSTFTLoss(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240]).to(dev),
        "gen_adv": losses.GeneratorAdversarialLoss(average_by_discriminators=False),
        "dis_adv": losses.DiscriminatorAdversarialLoss(average_by_discriminators=False),
    }
    opt_g = optimizers.FusedAdam(g.parameters(), lr=LR_G, betas=(0.5, 0.9), weight_decay=0.0)
    opt_d = optimizers.FusedAdam(d.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    # The discriminator phase scores the generator phase's output (update_prediction_after_generator_update=False), so
    # every loss of the step depends on the seeded inputs and weights only.  Regenerating after the update would make the
    # discriminator losses depend on that update, which the STFT adjoint's float atomics perturb (see below).
    step = GanTrainStep(g, d, crit, opt_g, opt_d, lambda_aux=1.0, lambda_adv=1.0, update_prediction_after_generator_update=False,
                        steps=1)
    corpus = datasets.DeviceCorpus(items, dev, hop_size=HOP)
    col = datasets.Collater(batch_max_steps=17920, hop_size=HOP, aux_context_window=0)
    np.random.seed(3)
    torch.manual_seed(3)
    x, y = col(corpus, [0, 1, 2])
    assert tuple(x[0].shape) == (3, 2, 56) and tuple(y.shape) == (3, 1, 17920)
    stats = step(x, y)
    torch.cuda.synchronize()
    return ({k: float(v) for k, v in stats.items()}, {k: p.grad.clone() for k, p in g.named_parameters()},
            {k: p.detach().clone() for k, p in g.named_parameters()})


def test_train_step_reproducible(dev):
    items = _items()
    s1, g1, p1 = _train_step(dev, items)
    s2, g2, p2 = _train_step(dev, items)
    for k in ("generator_loss", "spectral_convergence_loss", "log_stft_magnitude_loss", "adversarial_loss", "discriminator_loss",
              "real_loss", "fake_loss"):
        assert k in s1 and math.isfinite(s1[k]), (k, s1.get(k))
    # every loss is a forward of the seeded inputs and weights: bit-identical.  The gradients go through the STFT
    # adjoint's float atomics.
    for k in ("generator_loss", "spectral_convergence_loss", "log_stft_magnitude_loss", "adversarial_loss", "discriminator_loss",
              "real_loss", "fake_loss"):
        assert s1[k] == s2[k], (k, s1[k], s2[k])
    assert g1["emb.weight"].any() and g1["spk_emb.weight"].any()
    for k in g1:
        assert rel_l2(g1[k].cpu(), g2[k].cpu()) < 1e-4, k
        # Adam's first step moves each element by lr * m / (sqrt(v) + eps), at most lr: where a gradient near zero
        # changes sign between the runs, the two updates differ by up to 2 lr
        assert float((p1[k] - p2[k]).abs().max()) <= 2 * LR_G * (1 + 1e-3), k


def _units(n=5, seed=4, num_embs=100, num_spk=128):
    rng = np.random.RandomState(seed)
    return [np.stack([rng.randint(0, num_embs, size=T), np.full(T, rng.randint(0, num_spk))], axis=1)
            for T in (56, 100, 37, 112, 81)[:n]]


@pytest.mark.parametrize("rank,world", [(0, 1), (1, 2)])
def test_decoder_matches_inference(dev, rank, world):
    """Decoder.decode runs one inference per utterance of this rank's share: under the same seed it draws the same noise,
    so each waveform equals inference of that utterance alone, with and without PCM16 and with speaker ids."""
    from parallelwavegan_b200 import decode

    meta, _ = load_golden("dsym_style_vctk")
    m = _model(meta, dev)
    units = _units()
    mine = list(range(rank, len(units), world))
    dec = decode.Decoder(m, rank=rank, world=world)
    spk = [3, 0, 127, 9, 44]
    for kw in ({}, {"speakers": spk}):
        torch.manual_seed(5)
        with torch.no_grad():
            ref = {i: m.inference(torch.as_tensor(units[i][:, :1] if kw else units[i]).to(dev), g=spk[i] if kw else None)
                   for i in mine}
        torch.manual_seed(5)
        out = dec.decode(units, to_pcm16=False, **kw)
        assert sorted(out) == mine
        for i in mine:
            assert tuple(out[i].shape) == (len(units[i]) * 320, 1) and torch.equal(out[i], ref[i]), i
        torch.manual_seed(5)
        q = dec.decode([u[:, :1] for u in units] if kw else units, **kw)
        assert sorted(q) == mine
        for i in mine:
            assert q[i].dtype == np.int16 and np.array_equal(q[i], decode.pcm16(ref[i][:, 0]).cpu().numpy()), i
