"""StyleMelGAN generator (SURVEY.md 8 row a11b) on the libpwgb kernels vs the real-reference golden vectors and
the travelling oracle.

Tolerances.  The bar is 1e-3 relative L2.  The 9-block instance-normalised, softmax-gated stack is ill-conditioned
with the synthetic weights: on the CPU, in pure fp32, a 1e-6 relative perturbation of the conditioning moves the
reference output by 9e-5 rel-L2 and 1.9e-3 of peak at the worst sample, and the oracle differs from the reference
by 2.4e-5 / 5.3e-4 just through the order of fp32 sums.  Emulating the bf16x3 operand split of the tensor-core convs on
the CPU gives 2.5e-4 / 3.5e-3.
So the full-depth model is held to the 1e-3 rel-L2 bar and to 2e-2 of peak pointwise; single blocks and the small
model are held to 1e-3 on both."""
import json

import pytest
import torch
import torch.nn.functional as F

from helpers import golden_effective_weights, golden_weights, load_golden, max_abs_over_peak, rel_l2
from oracle import ref_ops, synth

pytestmark = pytest.mark.gpu
REL_TOL = 1e-3  # north_star bar


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


@pytest.mark.parametrize("T,C,slope", [(88, 64, 1.0), (1000, 32, 0.2), (7, 5, 1.0)])
def test_instance_norm(dev, T, C, slope):
    from parallelwavegan_b200 import ops

    x = synth.randn((2, C, T), 1) * 3.0 + 0.7
    ref = F.instance_norm(F.leaky_relu(x, slope) if slope != 1.0 else x)
    with torch.no_grad():
        y = ops.instance_norm(x.to(dev), pre_slope=slope)
    assert rel_l2(y.cpu(), ref) < 1e-5


@pytest.mark.parametrize("scale", [1, 2, 3])
def test_nearest_combine_gate(dev, scale):
    from parallelwavegan_b200 import ops

    B, C, T = 2, 24, 50
    xn = synth.randn((B, C, T), 2)
    cg = synth.randn((B, 2 * C, T * scale), 3)
    res = synth.randn((B, C, T), 4)
    up = lambda t: F.interpolate(t, scale_factor=scale, mode="nearest")
    with torch.no_grad():
        assert torch.equal(ops.upsample_nearest(xn.to(dev), scale).cpu(), up(xn))
        y = ops.tade_combine(cg.to(dev), xn.to(dev), scale)
        assert rel_l2(y.cpu(), cg[:, :C] * up(xn) + cg[:, C:]) < 1e-6
        for fn, gate in (("softmax", lambda t: torch.softmax(t, dim=1)), ("sigmoid", torch.sigmoid)):
            g = ops.tade_gate(cg.to(dev), res.to(dev), scale, fn)
            assert rel_l2(g.cpu(), gate(cg[:, :C]) * torch.tanh(cg[:, C:]) + up(res)) < 1e-5
            g0 = ops.tade_gate(cg.to(dev), None, 1, fn)
            assert rel_l2(g0.cpu(), gate(cg[:, :C]) * torch.tanh(cg[:, C:])) < 1e-5


@pytest.mark.parametrize("name", ["style_melgan_small", "style_melgan_v1"])
def test_style_melgan_generator_vs_reference(dev, name):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.StyleMelGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    m = m.eval().to(dev)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).to(dev)
    z = synth.randn(meta["z_shape"], meta["z_seed"]).to(dev)
    with torch.no_grad():
        x0 = m._noise_path(z)
        x1, c1 = m.blocks[0](x0, c)
        y = m(c, z)
    assert rel_l2(x0.cpu(), g["x0"]) < REL_TOL
    assert rel_l2(x1.cpu(), g["x1"]) < REL_TOL and rel_l2(c1.cpu(), g["c1"]) < REL_TOL
    assert tuple(y.shape) == tuple(g["y"].shape)
    deep = len(meta["kwargs"]["upsample_scales"]) > 4
    assert rel_l2(y.cpu(), g["y"]) < REL_TOL and max_abs_over_peak(y.cpu(), g["y"]) < (2e-2 if deep else REL_TOL)
    kw = meta["kwargs"]
    cfg = dict(kw, noise_upsample_negative_slope=kw["noise_upsample_activation_params"]["negative_slope"])
    ref = ref_ops.style_melgan_generator(golden_effective_weights(meta), c.cpu(), z.cpu(), cfg)
    assert rel_l2(y.cpu(), ref) < REL_TOL
    # weight norm removed: same function
    m.remove_weight_norm()
    with torch.no_grad():
        assert rel_l2(m(c, z).cpu(), g["y"]) < REL_TOL


def test_style_melgan_inference(dev):
    """inference() (style_melgan.py:226-262): noise length ceil(T / 88), conditioning replicate-padded, output cropped."""
    from parallelwavegan_b200 import models
    meta, _ = load_golden("style_melgan_v1")
    m = models.StyleMelGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    m = m.eval().to(dev)
    T = 100  # -> 2 noise frames, 176 conditioning frames after padding
    c = synth.randn((T, 80), 5)
    noise = synth.randn((1, 128, 2), 6)
    with torch.no_grad():
        y = m.inference(c.to(dev), noise=noise.to(dev))
    assert tuple(y.shape) == (T * 256, 1)
    cp = F.pad(c.t().unsqueeze(0), (0, 176 - T), mode="replicate")
    kw = meta["kwargs"]
    cfg = dict(kw, noise_upsample_negative_slope=0.2)
    ref = ref_ops.style_melgan_generator(golden_effective_weights(meta), cp, noise, cfg)[..., : T * 256]
    assert rel_l2(y.cpu(), ref.squeeze(0).t()) < REL_TOL


@pytest.mark.parametrize("scale", [1, 2, 3])
def test_tade_glue_gradients(dev, scale):
    """Adjoint kernels of InstanceNorm1d (with / without the fused LeakyReLU), nearest upsampling, the TADE modulation and
    the softmax / sigmoid gate with residual (layers/tade_res_block.py:52-160) vs torch autograd on the CPU."""
    from parallelwavegan_b200 import ops

    B, C, T = 2, 24, 50
    up = lambda t: F.interpolate(t, scale_factor=scale, mode="nearest")
    for slope in (1.0, 0.2):
        x = synth.randn((B, C, T), 11) * 2.0 + 0.3
        w = synth.randn((B, C, T), 12)
        xr = x.clone().requires_grad_(True)
        (F.instance_norm(F.leaky_relu(xr, slope) if slope != 1.0 else xr) * w).sum().backward()
        xd = x.clone().to(dev).requires_grad_(True)
        (ops.instance_norm(xd, pre_slope=slope) * w.to(dev)).sum().backward()
        assert rel_l2(xd.grad.cpu(), xr.grad) < 1e-4, slope
    xn, cg, res = synth.randn((B, C, T), 2), synth.randn((B, 2 * C, T * scale), 3), synth.randn((B, C, T), 4)
    w = synth.randn((B, C, T * scale), 5)
    xr, cr = xn.clone().requires_grad_(True), cg.clone().requires_grad_(True)
    ((cr[:, :C] * up(xr) + cr[:, C:]) * w).sum().backward()
    xd, cd = xn.clone().to(dev).requires_grad_(True), cg.clone().to(dev).requires_grad_(True)
    (ops.tade_combine(cd, xd, scale) * w.to(dev)).sum().backward()
    assert rel_l2(xd.grad.cpu(), xr.grad) < 1e-5 and rel_l2(cd.grad.cpu(), cr.grad) < 1e-5
    if scale > 1:
        xr = xn.clone().requires_grad_(True)
        (up(xr) * w).sum().backward()
        xd = xn.clone().to(dev).requires_grad_(True)
        (ops.upsample_nearest(xd, scale) * w.to(dev)).sum().backward()
        assert rel_l2(xd.grad.cpu(), xr.grad) < 1e-6
    for fn, gate in (("softmax", lambda t: torch.softmax(t, dim=1)), ("sigmoid", torch.sigmoid)):
        cr, rr = cg.clone().requires_grad_(True), res.clone().requires_grad_(True)
        ((gate(cr[:, :C]) * torch.tanh(cr[:, C:]) + up(rr)) * w).sum().backward()
        cd, rd = cg.clone().to(dev).requires_grad_(True), res.clone().to(dev).requires_grad_(True)
        (ops.tade_gate(cd, rd, scale, fn) * w.to(dev)).sum().backward()
        assert rel_l2(cd.grad.cpu(), cr.grad) < 1e-4, fn
        assert rel_l2(rd.grad.cpu(), rr.grad) < 1e-6, fn


def test_style_melgan_generator_gradients(dev):
    """StyleMelGAN generator training (row a11b): parameter and input gradients of the small golden model through the TADE
    adjoints, the tensor-core conv data / weight gradients and the transposed-conv noise path vs torch autograd through the
    CPU oracle, with the conditioning-aware bound (instance norm + softmax gates amplify fp32 rounding, see the header)."""
    from helpers import conditioning_tolerances
    from parallelwavegan_b200 import models

    meta, _ = load_golden("style_melgan_small")
    kw = json.loads(json.dumps(meta["kwargs"]))
    m = models.StyleMelGANGenerator(**kw)
    sd = golden_weights(meta)
    m.load_state_dict(sd, strict=True)
    c = synth.randn(meta["c_shape"], meta["c_seed"])
    z = synth.randn(meta["z_shape"], meta["z_seed"])
    cfg = dict(kw, noise_upsample_negative_slope=kw["noise_upsample_activation_params"]["negative_slope"])
    keep = {}

    def oracle(leaves):
        lf = {k: v.clone().requires_grad_(True) for k, v in leaves.items() if k != "__c"}
        cr = leaves["__c"].clone().requires_grad_(True)
        y = ref_ops.style_melgan_generator(ref_ops.fold_weight_norm(lf), cr, z, cfg)
        keep.setdefault("y", y.detach())
        keep.setdefault("t", synth.randn(tuple(y.shape), 77))
        (y * keep["t"]).sum().backward()
        out = {k: v.grad for k, v in lf.items()}
        out["__c"] = cr.grad
        return out

    ref, tol, obs = conditioning_tolerances(oracle, dict(sd, __c=c), rel_eps=2e-5)
    m = m.to(dev).train()
    cd = c.to(dev).requires_grad_(True)
    y = m(cd, z.to(dev))
    assert rel_l2(y.detach().cpu(), keep["y"]) < REL_TOL
    (y * keep["t"].to(dev)).sum().backward()
    bad = []
    for k, g in [("__c", cd.grad)] + [(k, p.grad) for k, p in m.named_parameters()]:
        e = rel_l2(g.cpu(), ref[k])
        if e >= tol[k]:
            bad.append((k, round(e, 5), round(tol[k], 5), round(obs[k], 6)))
    print("STYLE-GRAD loose bounds", [(k, round(t, 4)) for k, t in tol.items() if t > 1e-3][:6], "worst",
          max(rel_l2(p.grad.cpu(), ref[k]) for k, p in m.named_parameters()))
    assert not bad, bad[:10]
