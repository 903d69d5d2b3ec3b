"""VQ-VAE on the GPU: golden parity of forward / encode / decode, the nearest-code kernel against an fp64 brute force,
the decoder-input assembly bit for bit against torch.cat, its one-launch front end, NaN columns for out-of-range
indices, the backward kernels and the MSE mode against torch, every parameter's gradient against oracle autograd, one
vctk local_conditioned training step against the oracle step, and the conditioned collater."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import REL_TOL, conditioning_tolerances, load_golden, rel_l2
from oracle import ref_optim, ref_ops, ref_vqvae, synth
from test_vqvae_cpu import vq_weights

pytestmark = pytest.mark.gpu
NAMES = ["vqvae_yesno", "vqvae_vctk_g", "vqvae_vctk_lg"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _model(meta, dev):
    from parallelwavegan_b200 import models

    m = models.VQVAE(**copy.deepcopy(meta["kwargs"]))
    m.load_state_dict(vq_weights(meta, fold=False))
    return m.to(dev).eval()


def _cond(g, dev):
    return (g["l"].to(dev) if "l" in g else None), (g["g"].to(dev) if "g" in g else None)


@pytest.mark.parametrize("name", NAMES)
def test_golden_parity(dev, name):
    meta, g = load_golden(name)
    m = _model(meta, dev)
    l, gid = _cond(g, dev)
    x = g["x"].to(dev)
    for _ in range(2):  # with weight norm, then folded
        with torch.no_grad():
            x_bar, z_e, z_q = m(x, l, gid)
            idx = m.encode(x)
            dec = m.decode(idx, l, gid)
        assert torch.equal(idx.cpu(), g["indices"])
        for a, b in ((x_bar, g["x_bar"]), (z_e, g["z_e"]), (z_q, g["z_q"]), (dec, g["decode"])):
            assert tuple(a.shape) == tuple(b.shape) and rel_l2(a.cpu(), b) < REL_TOL
        m.remove_weight_norm()


def _fp64_dist(z, cb):
    x = z.double().transpose(1, 2).reshape(-1, cb.shape[1])
    c = cb.double()
    return (c * c).sum(1)[None] + (x * x).sum(1)[:, None] - 2 * x @ c.t(), x


@pytest.mark.parametrize("D", [8, 100, 256])
@pytest.mark.parametrize("K", [16, 500, 512])
def test_nearest_code_against_fp64(dev, D, K):
    from parallelwavegan_b200 import ops

    torch.manual_seed(D * 1000 + K)
    for B, T in ((2, 45), (1, 1), (3, 70), (0, 9)):
        z = torch.randn(B, D, T)
        cb = torch.randn(K, D) * 0.8
        idx, zq, _ = ops.vq_raw(z.to(dev), cb.to(dev), z_q=True, dec=False)
        idx2, _, _ = ops.vq_raw(z.to(dev), cb.to(dev), z_q=False, dec=False)
        assert torch.equal(idx, idx2) and tuple(idx.shape) == (B, T)
        if B == 0:
            continue
        d, x = _fp64_dist(z, cb)
        chosen = d.gather(1, idx.cpu().reshape(-1, 1)).squeeze(1)
        best, arg = d.min(1)
        # fp32 rounding of (|c|^2 + |x|^2) - 2 x.c: a few ulps of the terms' magnitude, D-term sums
        bound = 4 * D * 2.0**-24 * ((x * x).sum(1) + (cb.double() ** 2).sum(1).max())
        assert bool((chosen - best <= bound).all())
        s = d.sort(1)[0]
        clear = (s[:, 1] - s[:, 0]) > bound
        assert bool(clear.any()) and torch.equal(idx.cpu().reshape(-1)[clear], arg[clear])
        assert torch.equal(zq.cpu(), cb[idx.cpu()].permute(0, 2, 1))


def test_ties_nan_and_determinism(dev):
    from parallelwavegan_b200 import ops

    torch.manual_seed(3)
    D, K = 64, 300
    cb = torch.randn(K, D)
    cb[250] = cb[7]  # duplicated rows: the lower index wins
    cb[299] = cb[41]
    z = torch.randn(2, D, 40)
    z[0, :, 3] = cb[7]
    z[1, :, 5] = cb[41]
    z[1, 7, 9] = float("nan")  # every distance NaN: torch.min takes the first NaN, index 0
    idx, _, _ = ops.vq_raw(z.to(dev), cb.to(dev), z_q=False, dec=False)
    assert int(idx[0, 3]) == 7 and int(idx[1, 5]) == 41 and int(idx[1, 9]) == 0
    d = ref_vqvae.distances(z, cb)
    assert int(d.min(1)[1].reshape(2, 40)[1, 9]) == 0  # torch.min agrees
    cbn = cb.clone()
    cbn[100, 0] = float("nan")  # one NaN code: it wins every frame
    idx_n, _, _ = ops.vq_raw(z.to(dev), cbn.to(dev), z_q=False, dec=False)
    assert bool((idx_n.cpu() == ref_vqvae.distances(z, cbn).min(1)[1].reshape(2, 40)).all())
    a = ops.vq_raw(z.to(dev), cb.to(dev))
    b = ops.vq_raw(z.to(dev), cb.to(dev))
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])


def test_assembly_bit_identical_and_nan_columns(dev):
    from parallelwavegan_b200 import ops

    torch.manual_seed(4)
    B, D, T, K, Cl, Cg, ng = 3, 256, 77, 512, 32, 128, 10
    z, cb = torch.randn(B, D, T), torch.randn(K, D) * 0.5
    l, gt = torch.randn(B, Cl, T), torch.randn(ng, Cg)
    g = torch.tensor([4, 0, 9])
    idx, zq, dec = ops.vq_raw(z.to(dev), cb.to(dev), l=l.to(dev), global_table=gt.to(dev), g=g.to(dev))
    codes = cb[idx.cpu()].permute(0, 2, 1)
    ref = torch.cat([codes, l, gt[g].unsqueeze(2).expand(-1, -1, T)], dim=1)
    assert torch.equal(dec.cpu(), ref) and torch.equal(zq.cpu(), codes)
    for lc, gc in ((l, None), (None, g)):  # one condition at a time
        _, _, dec1 = ops.vq_raw(None, cb.to(dev), indices=idx, l=lc.to(dev) if lc is not None else None,
                                global_table=gt.to(dev) if gc is not None else None, g=gc.to(dev) if gc is not None else None)
        parts = [codes] + ([lc] if lc is not None else []) + ([gt[gc].unsqueeze(2).expand(-1, -1, T)] if gc is not None else [])
        assert torch.equal(dec1.cpu(), torch.cat(parts, 1))
    bad = idx.clone()
    bad[0, 5], bad[2, 70] = K, -1
    _, _, decb = ops.vq_raw(None, cb.to(dev), indices=bad, l=l.to(dev), global_table=gt.to(dev),
                            g=torch.tensor([4, 10, 9]).to(dev))
    decb = decb.cpu()
    assert bool(decb[0, :, 5].isnan().all()) and bool(decb[2, :, 70].isnan().all()) and bool(decb[1].isnan().all())
    keep = torch.ones(B, T, dtype=torch.bool)
    keep[0, 5] = keep[2, 70] = False
    keep[1] = False
    assert torch.equal(decb.permute(0, 2, 1)[keep], ref.permute(0, 2, 1)[keep])


def test_front_end_is_one_launch(dev):
    """Search, gather and assembly of the eval forward are one launch: VQVAE = encoder + local_embed + VQ + decoder."""
    from parallelwavegan_b200 import capi, ops

    meta, g = load_golden("vqvae_vctk_lg")
    m = _model(meta, dev)
    l, gid = _cond(g, dev)
    x = g["x"].to(dev)
    with torch.no_grad():
        m(x, l, gid)
        torch.cuda.synchronize()
        capi.reset_launch_count()
        m(x, l, gid)
        torch.cuda.synchronize()
        n_all = capi.launch_count()
        z_e = m.encoder(x)[-1]
        le = m._local(l)
        _, _, dec = ops.vq_raw(z_e, m.codebook.embedding.weight, z_q=True, l=le, global_table=m.global_embed.weight, g=gid)
        torch.cuda.synchronize()
        capi.reset_launch_count()
        m.encoder(x)
        m._local(l)
        m.decoder(dec)
        torch.cuda.synchronize()
        n_rest = capi.launch_count()
        capi.reset_launch_count()
        ops.vq_raw(z_e, m.codebook.embedding.weight, z_q=True, l=le, global_table=m.global_embed.weight, g=gid)
        torch.cuda.synchronize()
        assert capi.launch_count() == 1
    assert n_all == n_rest + 1, (n_all, n_rest)


def test_backward_kernels(dev):
    from parallelwavegan_b200 import ops

    torch.manual_seed(5)
    B, D, T, K, Cl, Cg, ng = 4, 64, 50, 40, 8, 16, 6
    z = torch.randn(B, D, T, device=dev, requires_grad=True)
    cb = (torch.randn(K, D) * 0.5).to(dev).requires_grad_(True)
    l = torch.randn(B, Cl, T, device=dev, requires_grad=True)
    gt = torch.randn(ng, Cg, device=dev, requires_grad=True)
    g = torch.tensor([2, 5, 2, 0], device=dev)
    dec, zq, idx = ops.vq(z, cb, l=l, global_table=gt, g=g)
    gd, gq = torch.randn_like(dec), torch.randn_like(zq)
    grads = torch.autograd.grad((dec * gd).sum() + (zq * gq).sum(), [z, cb, l, gt])
    grads2 = torch.autograd.grad(sum((t * w).sum() for t, w in zip(ops.vq(z, cb, l=l, global_table=gt, g=g)[:2], (gd, gq))),
                                 [z, cb, l, gt])
    for a, b in zip(grads, grads2):
        assert torch.equal(a, b)  # run to run
    assert torch.equal(grads[0], gd[:, :D]) and torch.equal(grads[2], gd[:, D : D + Cl])
    ic = idx.cpu().reshape(-1)
    ref_cb = torch.zeros(K, D, dtype=torch.float64).index_add_(0, ic, gq.cpu().double().permute(0, 2, 1).reshape(-1, D))
    assert rel_l2(grads[1].cpu(), ref_cb) < 1e-6
    gsum = gd[:, D + Cl :].cpu().double().sum(2)
    ref_gt = torch.zeros(ng, Cg, dtype=torch.float64).index_add_(0, g.cpu(), gsum)
    assert rel_l2(grads[3].cpu(), ref_gt) < 1e-6
    # the functions-module mirror: the codes' gradient reaches both the inputs and the codebook
    from parallelwavegan_b200.functions import vector_quantize, vector_quantize_straight_through

    zt = z.detach().transpose(1, 2).requires_grad_(True)
    codes, flat = vector_quantize_straight_through(zt, cb)
    assert torch.equal(flat, idx.reshape(-1)) and torch.equal(vector_quantize(zt, cb), idx)
    gc = torch.randn_like(codes)
    gz, gcb = torch.autograd.grad((codes * gc).sum(), [zt, cb])
    assert torch.equal(gz, gc)
    ref_cb = torch.zeros(K, D, dtype=torch.float64).index_add_(0, ic, gc.cpu().double().reshape(-1, D))
    assert rel_l2(gcb.cpu(), ref_cb) < 1e-6


def test_mse_mode(dev):
    from parallelwavegan_b200 import losses

    torch.manual_seed(6)
    x = torch.randn(3, 256, 37, device=dev, requires_grad=True)
    y = torch.randn(3, 256, 37, device=dev, requires_grad=True)
    out = losses.MSELoss()(x, y)
    ref = F.mse_loss(x.detach().double(), y.detach().double())
    assert abs(float(out) - float(ref)) <= 1e-6 * float(ref)
    gx, gy = torch.autograd.grad(out * 3.0, [x, y])
    rx = 3.0 * 2 * (x.detach() - y.detach()) / x.numel()
    assert rel_l2(gx, rx) < 1e-6 and rel_l2(gy, -rx) < 1e-6


def test_parameter_gradients_against_oracle(dev):
    meta, g = load_golden("vqvae_vctk_lg")
    cfg = meta["kwargs"]
    sd = vq_weights(meta, fold=False)
    x, l, gid = g["x"], g["l"], g["g"]
    gout = synth.randn(tuple(g["x_bar"].shape), 31)
    gzq = synth.randn(tuple(g["z_q"].shape), 32, 0.1)
    gze = synth.randn(tuple(g["z_e"].shape), 33, 0.1)
    keep = {}

    def oracle(leaves):
        leaf = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
        x_bar, z_e, z_q, idx = ref_vqvae.vqvae_forward(ref_ops.fold_weight_norm(leaf), x, cfg, l, gid)
        ((x_bar * gout).sum() + (z_q * gzq).sum() + (z_e * gze).sum()).backward()
        keep.setdefault("idx", idx)
        return {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaf.items()}

    ref, tol, obs = conditioning_tolerances(oracle, dict(sd))
    assert torch.equal(keep["idx"], g["indices"])
    m = _model(meta, dev).train()
    x_bar, z_e, z_q = m(x.to(dev), l.to(dev), gid.to(dev))
    ((x_bar * gout.to(dev)).sum() + (z_q * gzq.to(dev)).sum() + (z_e * gze.to(dev)).sum()).backward()
    names = [k for k, _ in m.named_parameters()]
    for part in ("encoder.", "codebook.", "local_embed.", "global_embed.", "decoder."):
        assert any(k.startswith(part) for k in names), part
    bad = [(k, rel_l2(p.grad.cpu(), ref[k]), tol[k]) for k, p in m.named_parameters() if rel_l2(p.grad.cpu(), ref[k]) >= tol[k]]
    assert not bad, bad


def _vq_items(n=4):
    items = []
    for k in range(n):
        frames = 40 + 9 * k
        items.append((synth.randn((frames * 64,), 9000 + k, 0.3).numpy(), synth.randn((frames, 2), 9100 + k).numpy(),
                      np.array([k % 3 * 5], dtype=np.int64)))
    return items


def test_conditioned_collater_matches_oracle(dev):
    from parallelwavegan_b200 import datasets

    items = _vq_items()
    items[1] = (items[1][0][:-20], items[1][1], items[1][2])  # edge-padded by _adjust_length
    for local in (True, False):
        its = items if local else [(x, gid) for x, _, gid in items]
        corpus = datasets.DeviceCorpus(its, dev, hop_size=64 if local else None, global_condition=True)
        col = datasets.Collater(batch_max_steps=2048, hop_size=64, aux_context_window=0, use_aux_input=False,
                                use_global_condition=True, use_local_condition=local)
        np.random.seed(17)
        (l, gg), y = col(corpus, [0, 1, 2, 3])
        np.random.seed(17)
        (lr, gr), yr = ref_vqvae.collate_vq(its, 2048, 64, 0, use_local_condition=local, use_global_condition=True)
        assert torch.equal(y.cpu(), torch.from_numpy(yr)) and torch.equal(gg.cpu(), torch.from_numpy(gr))
        assert (l is None and lr is None) or torch.equal(l.cpu(), torch.from_numpy(lr))


STFT = dict(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240])
LAMBDA = dict(lambda_aux=1.0, lambda_adv=4.0, lambda_feat_match=25.0, lambda_commit=0.25)  # local_conditioned_melgan_vae.v3


def _vctk_step(dev, meta, dsd, l, gid, y):
    from parallelwavegan_b200 import losses, models, optimizers
    from parallelwavegan_b200.train_step import GanTrainStep

    gm = _model(meta, dev).train()
    d = models.MelGANMultiScaleDiscriminator()
    d.load_state_dict(dsd)
    d = d.to(dev).train()
    crit = {"stft": losses.MultiResolutionSTFTLoss(**STFT).to(dev), "mse": losses.MSELoss(),
            "gen_adv": losses.GeneratorAdversarialLoss(), "dis_adv": losses.DiscriminatorAdversarialLoss(),
            "feat_match": losses.FeatureMatchLoss()}
    opt_g = optimizers.FusedAdam(gm.parameters(), lr=1e-4, eps=1e-6)
    opt_d = optimizers.FusedAdam(d.parameters(), lr=5e-5, eps=1e-6)
    step = GanTrainStep(gm, d, crit, opt_g, opt_d, lambda_aux=LAMBDA["lambda_aux"], lambda_adv=LAMBDA["lambda_adv"],
                        lambda_feat_match=LAMBDA["lambda_feat_match"], lambda_commit=LAMBDA["lambda_commit"], grad_norm_g=10,
                        grad_norm_d=1, steps=1)
    stats = step((l.to(dev), gid.to(dev)), y.to(dev))
    torch.cuda.synchronize()
    return {k: float(v) for k, v in stats.items()}, {k: p.detach().cpu().clone() for k, p in gm.named_parameters()}


def _adam(params, grads, lr, eps, max_norm):
    _, c = ref_optim.clip_coef(list(grads.values()), max_norm)
    out = {}
    for k, p in params.items():
        q = p.clone()
        ref_optim.adam_step(q, grads[k] * c, torch.zeros_like(q), torch.zeros_like(q), 1, lr, (0.9, 0.999), eps, 0.0)
        out[k] = q
    return out


def test_vctk_train_step_against_oracle(dev):
    """One GanTrainStep of egs/vctk/vq1/conf/local_conditioned_melgan_vae.v3.yaml with the discriminator on (batch of 2,
    2048 samples): loss scalars vs the oracle step, generator parameters after the fused Adam step vs the oracle update,
    and two runs bit-identical in the generator phase (every loss computed before the first backward); the generator's
    gradients then pass the STFT loss adjoint's float atomics, so the parameters agree to rounding only."""
    from parallelwavegan_b200 import models

    meta, _ = load_golden("vqvae_vctk_lg")
    cfg = meta["kwargs"]
    sd = vq_weights(meta, fold=False)
    dspec = [(k, tuple(v.shape)) for k, v in models.MelGANMultiScaleDiscriminator().state_dict().items()]
    dsd = synth.synth_state_dict(dspec, 61, 1.3)
    y = synth.randn((2, 1, 2048), 62, 0.3)
    l = synth.randn((2, 2, 32), 63)
    gid = torch.tensor([5, 77])
    s1, p1 = _vctk_step(dev, meta, dsd, l, gid, y)
    s2, p2 = _vctk_step(dev, meta, dsd, l, gid, y)

    # ---- oracle: generator phase with autograd, Adam with clipping, discriminator phase on the updated generator
    lg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    wd = ref_ops.fold_weight_norm(dsd)
    x_bar, z_e, z_q, _ = ref_vqvae.vqvae_forward(ref_ops.fold_weight_norm(lg), y, cfg, l, gid)
    quant, commit = ref_vqvae.vq_losses(z_e, z_q)
    sc, mag = ref_ops.mr_stft_loss(x_bar, y, **{k: tuple(v) for k, v in STFT.items()})
    p_hat = ref_ops.melgan_msd(wd, x_bar)
    with torch.no_grad():
        p_real = ref_ops.melgan_msd(wd, y)
    adv = ref_ops.generator_adv_loss(p_hat)
    fm = ref_ops.feature_match_loss(p_hat, p_real)
    gen = (quant + LAMBDA["lambda_commit"] * commit + sc + mag) * LAMBDA["lambda_aux"] + LAMBDA["lambda_adv"] * (adv + LAMBDA["lambda_feat_match"] * fm)
    gen.backward()
    new = _adam(sd, {k: v.grad for k, v in lg.items()}, 1e-4, 1e-6, 10.0)
    with torch.no_grad():
        # the discriminator phase from the generator this step left: Adam's first update is lr * sign(g), so elements whose
        # gradient is within rounding of zero may step either way, and the regenerated audio follows them
        x_bar2, _, _, _ = ref_vqvae.vqvae_forward(ref_ops.fold_weight_norm(p1), y, cfg, l, gid)
        real, fake = ref_ops.discriminator_adv_loss(ref_ops.melgan_msd(wd, x_bar2), ref_ops.melgan_msd(wd, y))
    ref = dict(quantization_loss=quant, commitment_loss=commit, spectral_convergence_loss=sc, log_stft_magnitude_loss=mag,
               adversarial_loss=adv, feature_matching_loss=fm, generator_loss=gen, real_loss=real, fake_loss=fake,
               discriminator_loss=real + fake)
    for k, r in ref.items():
        r = float(r)
        assert abs(s1[k] - r) <= 1e-4 * abs(r), (k, s1[k], r)
    bad = [(k, rel_l2(p1[k], new[k])) for k in new if rel_l2(p1[k], new[k]) >= 1e-3]
    assert not bad, bad
    for k in ("generator_loss", "quantization_loss", "commitment_loss", "adversarial_loss", "feature_matching_loss"):
        assert s1[k] == s2[k], (k, s1[k], s2[k])
    for k in p1:
        assert rel_l2(p1[k], p2[k]) < 1e-4, k
