"""Bring-up probe for the tensor-core conv path: prints error statistics for several shapes and
descriptor variants, never asserts (diagnostics for a box without interactive access)."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

import __graft_entry__

__graft_entry__.build()
from parallelwavegan_b200 import capi, ops

dev = torch.device("cuda:0")
L = capi.lib()
L.pwgb_debug_set.argtypes = [C.c_int, C.c_int]
shapes = [(32, 16, 1, 1, 128, 1), (32, 32, 3, 1, 300, 2), (64, 64, 7, 3, 1000, 2), (256, 256, 3, 1, 513, 1), (128, 128, 11, 5, 700, 2)]
variants = [int(v) for v in (sys.argv[1:] or ["0"])]
for variant in variants:
    L.pwgb_debug_set(1, variant)
    for (cin, cout, k, dil, T, B) in shapes:
        torch.manual_seed(0)
        pad = (k - 1) // 2 * dil
        x = torch.randn(B, cin, T)
        w = torch.randn(cout, cin, k) / (cin * k) ** 0.5
        ref = F.conv1d(x, w, None, padding=pad, dilation=dil)
        ops.ENGINE = "auto"
        try:
            y = ops.conv1d(x.to(dev), w.to(dev), None, padding=pad, dilation=dil)
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            print(f"variant {variant} shape {(cin, cout, k, dil, T, B)}: EXC {e}")
            break
        y = y.cpu()
        err = float((y - ref).norm() / ref.norm())
        # diagnostics: which rows/cols are wrong
        bad = ((y - ref).abs() > 1e-3 * ref.abs().max())
        print(f"variant {variant} shape {(cin, cout, k, dil, T, B)}: rel {err:.3e} bad frac {bad.float().mean():.3f} "
              f"nan {int(torch.isnan(y).sum())} | y[0,0,:4] {y[0,0,:4].tolist()} ref {ref[0,0,:4].tolist()}")
        if err > 1e-3:
            bt = bad[0].float().mean(0)  # per time
            bc = bad[0].float().mean(1)  # per channel
            print("   bad per-channel (first 32):", [round(float(v), 2) for v in bc[:32]])
            print("   bad per-time (first 40):", [round(float(v), 2) for v in bt[:40]])
            # ratio test
            print("   y/ref sample:", [(round(float(y[0, c, t]), 4), round(float(ref[0, c, t]), 4)) for c in (0, 1, 8, 15) for t in (0, 1, 7, 8, 64, 127) if c < cout and t < T])
