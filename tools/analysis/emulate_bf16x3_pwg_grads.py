import os, sys, json; _R = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..'); sys.path.insert(0, os.path.join(_R, 'tests')); sys.path.insert(0, _R)
import torch, torch.nn.functional as F
from helpers import rel_l2
from oracle import ref_ops, synth
from parallelwavegan_b200 import models
torch.set_num_threads(8)
kw = dict(in_channels=1, out_channels=1, kernel_size=3, layers=6, stacks=3, residual_channels=64, gate_channels=128,
          skip_channels=64, aux_channels=80, aux_context_window=2, dropout=0.0, use_weight_norm=True,
          upsample_conditional_features=True, upsample_net="ConvInUpsampleNetwork", upsample_params={"upsample_scales": [4, 4, 4, 4]})
g = models.ParallelWaveGANGenerator(**json.loads(json.dumps(kw)))
sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 51, 1.0)
B, frames = 2, 12
c = synth.randn((B, 80, frames + 4), 53); z = synth.randn((B, 1, frames * 256), 54); y = synth.randn((B, 1, frames * 256), 55, 0.3)
cfg = dict(kw, upsample_scales=[4, 4, 4, 4])
orig=F.conv1d
def split(t):
    h=t.to(torch.bfloat16).to(torch.float32); l=(t-h).to(torch.bfloat16).to(torch.float32); return h,l
def make_conv(ragged_ok):
    def conv3(x, wt, b=None, **k):
        cin=wt.shape[1]; cout=wt.shape[0]
        ok = k.get("groups",1)==1 and cout % 16 == 0 and (cin % 32 == 0 or (ragged_ok and cin >= 32))
        if ok:
            xh,_=split(x.detach()); xq=x+(xh-x).detach(); xl=(x-xq).detach(); xl=split(xl)[0]
            wh,_=split(wt.detach()); wq=wt+(wh-wt).detach(); wl=split((wt-wq).detach())[0]
            yv=orig(xq,wq,None,**k)+orig(xl,wq.detach(),None,**k)+orig(xq.detach(),wl,None,**k)
            return yv if b is None else yv+b[None,:,None]
        return orig(x,wt,b,**k)
    return conv3
names=[k for k in sd]
def run(conv):
    F.conv1d=conv
    leaf={k:v.clone().requires_grad_(True) for k,v in sd.items()}
    yr=ref_ops.pwg_generator(ref_ops.fold_weight_norm(leaf), z, c, cfg)
    sc,mag=ref_ops.mr_stft_loss(yr.squeeze(1), y.squeeze(1))
    gs=torch.autograd.grad(sc+mag,[leaf[k] for k in names],allow_unused=True)
    F.conv1d=orig
    return yr.detach(), {k:v for k,v in zip(names,gs) if v is not None}
y0,g0=run(orig)
for name,ragged in (("v13",False),("v14 ragged",True)):
    y1,g1=run(make_conv(ragged))
    errs={k:rel_l2(g1[k],g0[k]) for k in g0 if float(g0[k].abs().max())>1e-6}
    worst=sorted(errs.items(), key=lambda kv:-kv[1])[:6]
    print(name,"fwd rel",rel_l2(y1,y0),[(k,round(v,4)) for k,v in worst])
    print("   up_layers:",[(k,round(errs[k],4), float(g0[k].flatten()[0])) for k in errs if "up_layers" in k and k.endswith("weight_g")])
