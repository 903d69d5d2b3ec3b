import os, sys; _R = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..'); sys.path.insert(0, os.path.join(_R, 'tests')); sys.path.insert(0, _R)
import torch, torch.nn.functional as F
from helpers import rel_l2
from oracle import ref_ops, synth
from parallelwavegan_b200 import models
torch.set_num_threads(8)
kw = dict(in_channels=80, out_channels=1, channels=64, kernel_size=7, upsample_scales=[8, 4, 2],
          upsample_kernel_sizes=[16, 8, 4], resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3, 5], [1, 3]], use_causal_conv=True)
g = models.HiFiGANGenerator(**kw)
sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 17, 1.15)
c = synth.randn((2, 80, 32), 23); y = synth.randn((2, 1, 32 * 64), 24, 0.3)
melmat = torch.from_numpy(ref_ops.slaney_mel_filterbank(22050, 1024, 80, 0, 11025).T.copy())
orig=F.conv1d
def split(t):
    h=t.to(torch.bfloat16).to(torch.float32); l=(t-h).to(torch.bfloat16).to(torch.float32); return h,l
def make_conv(ragged_ok):
    def conv3(x, wt, b=None, **k):
        cin=wt.shape[1]; cout=wt.shape[0]
        ok = cout % 16 == 0 and (cin % 32 == 0 or (ragged_ok and cin >= 32))
        if ok:
            xh,xl=split(x.detach()); xh=x+(xh-x).detach(); xl=(x-xh).detach()*0+xl  # straight-through: gradient as fp32
            wh,wl=split(wt.detach()); whh=wt+(wh-wt).detach()
            yv=orig(xh,whh,None,**k)+orig(xl,whh.detach(),None,**k)+orig(xh.detach(),wl,None,**k)
            return yv if b is None else yv+b[None,:,None]
        return orig(x,wt,b,**k)
    return conv3
def grads(conv):
    F.conv1d=conv
    leaf={k:v.clone().requires_grad_(True) for k,v in sd.items()}
    cr=c.clone().requires_grad_(True)
    yr=ref_ops.hifigan_generator(ref_ops.fold_weight_norm(leaf), cr, dict(kw, negative_slope=0.1))
    ref_ops.mel_loss(yr, y, melmat, log_base=None).backward()
    F.conv1d=orig
    return yr.detach(), {k:v.grad for k,v in leaf.items()}, cr.grad
y0,g0,c0=grads(orig)
for name,ragged in (("v13 (input conv exact)",False),("v14 (input conv bf16x3)",True)):
    y1,g1,c1=grads(make_conv(ragged))
    errs={k:rel_l2(g1[k],g0[k]) for k in g0 if g0[k] is not None}
    worst=sorted(errs.items(), key=lambda kv:-kv[1])[:5]
    print(name, "fwd rel", rel_l2(y1,y0), "dc", rel_l2(c1,c0), "worst grads", [(k,round(v,5)) for k,v in worst])

# conditioning-aware criterion for weight-norm pairs: |a - r| relative to ||dL/dw_eff||,
# ||dL/dw||^2 = (dL/dg)^2 + (||v|| / g)^2 ||dL/dv||^2  (per output channel, summed)
def wn_scale(gr, sd_, name_g):
    name_v = name_g[:-2] + "_v"
    v, gg = sd_[name_v], sd_[name_g]
    dims = tuple(range(1, v.dim()))
    vn = v.pow(2).sum(dim=dims, keepdim=True).sqrt()
    dv = gr[name_v]
    return float(((gr[name_g] ** 2).sum() + ((vn / gg) ** 2 * dv.pow(2)).sum()).sqrt())
y1, g1, c1 = grads(make_conv(True))
rows = []
for k in g0:
    if g0[k] is None or not (k.endswith("weight_g") or k.endswith("weight_v")):
        continue
    kg = k if k.endswith("_g") else k[:-2] + "_g"
    sc = wn_scale(g0, sd, kg)
    if k.endswith("_v"):
        v, gg = sd[k], sd[kg]
        sc = sc * float((gg / v.pow(2).sum(dim=tuple(range(1, v.dim())), keepdim=True).sqrt()).abs().max())
    rows.append((float((g1[k] - g0[k]).norm()) / sc, rel_l2(g1[k], g0[k]), k))
rows.sort(reverse=True)
print("v14 emulation, error / ||dL/dw_eff|| (first column) vs plain rel-L2:")
for r in rows[:6]:
    print("  %.5f  %.5f  %s" % r)
