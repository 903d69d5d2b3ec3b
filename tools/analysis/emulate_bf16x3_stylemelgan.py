import os, sys; _R = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..'); sys.path.insert(0, os.path.join(_R, 'tests')); sys.path.insert(0, _R)
import torch, torch.nn.functional as F
from helpers import golden_effective_weights, load_golden, rel_l2, max_abs_over_peak
from oracle import ref_ops, synth
torch.set_num_threads(8)
meta,g=load_golden("style_melgan_v1")
w=golden_effective_weights(meta); kw=meta["kwargs"]
cfg=dict(kw, noise_upsample_negative_slope=0.2)
c=synth.randn(meta["c_shape"], meta["c_seed"]); z=synth.randn(meta["z_shape"], meta["z_seed"])
y_fp32=ref_ops.style_melgan_generator(w,c,z,cfg)
print("oracle vs golden: rel", rel_l2(y_fp32,g["y"]), "max/peak", max_abs_over_peak(y_fp32,g["y"]))
# emulate bf16x3 convs: x = xh + xl, w = wh + wl ; y = xh*wh + xl*wh + xh*wl (fp32 accumulate)
def split(t):
    h=t.to(torch.bfloat16).to(torch.float32); l=(t-h).to(torch.bfloat16).to(torch.float32); return h,l
orig_conv=F.conv1d
def conv3(x, wt, b=None, **k):
    cin=wt.shape[1]; cout=wt.shape[0]
    if cin % 32 == 0 and cout % 16 == 0:   # tensor-core path condition
        xh,xl=split(x); wh,wl=split(wt)
        y=orig_conv(xh,wh,None,**k)+orig_conv(xl,wh,None,**k)+orig_conv(xh,wl,None,**k)
        return y if b is None else y+b[None,:,None]
    return orig_conv(x,wt,b,**k)
F.conv1d=conv3
y_e=ref_ops.style_melgan_generator(w,c,z,cfg)
F.conv1d=orig_conv
print("bf16x3 emulation vs fp32 oracle: rel", rel_l2(y_e,y_fp32), "max/peak", max_abs_over_peak(y_e,y_fp32))
d=(y_e-y_fp32).abs().flatten(); print("err quantiles", [float(d.quantile(q)) for q in (0.5,0.9,0.99,0.999)], float(d.max()), "peak", float(y_fp32.abs().max()))
# perturbation sensitivity: pure fp32 noise of 1e-6 relative on the input conditioning
y_p=ref_ops.style_melgan_generator(w,c*(1+1e-6*torch.randn_like(c)),z,cfg)
print("1e-6 input perturbation: rel", rel_l2(y_p,y_fp32), "max/peak", max_abs_over_peak(y_p,y_fp32))
