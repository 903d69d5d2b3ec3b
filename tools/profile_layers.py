"""Per-launch table of the HiFi-GAN v1 C2 forward (CUDA events on the launching stream).  For conv1d_tc launches the
last column is the tile plan: MT (64-row blocks per warpgroup), na / nb / ns (operand buffers, weight stages, raw
activation stages) and whether the epilogue went through the shared-memory tile (staged) or registers.  For fused ResBlock
pairs (resblock_pair_tc) it is the output / conv rows per tile, conv1 operand buffers, weight stages of both rings and
raw stages.  For the 128- and 256-channel pairs (resblock_pair_packed_tc: conv1 and conv2 with the packed intermediate
between them) it is conv2's conv1d_tc plan."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from parallelwavegan_b200 import capi, ops

model, _ = bench.synth_weights()
dev = torch.device("cuda:0")
model = model.to(dev)
mel = torch.randn(bench.BATCH, 80, bench.FRAMES, device=dev)

plans = {}
_done = ops._Prof.done


def _done_with_plan(self):
    _done(self)
    if ops.PROFILE is not None and self.name in ("conv1d_tc", "resblock_pair_packed_tc"):
        v = (C.c_int * 5)()
        if capi.lib().pwgb_debug_get(1, C.cast(v, C.c_void_p), C.sizeof(v)) == 0:
            plans[len(ops.PROFILE) - 1] = f"MT{v[0]} na{v[1]} nb{v[2]} ns{v[3]} {'staged' if v[4] else 'reg'}"
    elif ops.PROFILE is not None and self.name == "resblock_pair_tc":
        # desc "B.. C.. k.. d.. T..": the plan is a function of the shape
        f = {s[0]: int(s[1:]) for s in self.desc.split()}
        pl = ops.resblock_pair_plan(f["C"], f["T"], f["k"], f["d"], batch=f["B"])
        plans[len(ops.PROFILE) - 1] = f"rows {pl['M2']}/{pl['TT']} na{pl['na']} nb{pl['nb']} ns{pl['ns']}"


ops._Prof.done = _done_with_plan
with torch.no_grad():
    for _ in range(3):
        model(mel)
    torch.cuda.synchronize()
    ops.PROFILE = []
    model(mel)
    torch.cuda.synchronize()
prof, ops.PROFILE = ops.PROFILE, None
tot = 0.0
print(f"{'kernel':18s} {'shape':46s} {'ms':>8s} {'TFLOP/s':>8s} {'algGB/s':>8s}  plan")
for i, (name, fl, by, a, b, desc) in enumerate(prof):
    ms = a.elapsed_time(b)
    tot += ms
    print(f"{name:18s} {desc:46s} {ms:8.3f} {fl / ms / 1e9:8.1f} {by / ms / 1e6:8.0f}  {plans.get(i, '')}")
print("total ms", tot)
