"""Run single representative conv launches (for ncu captures): args = list of 'cin,k,d,T,B'."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from parallelwavegan_b200 import ops

dev = torch.device("cuda:0")
if os.environ.get("PWGB_TC_VARIANT"):
    from parallelwavegan_b200 import capi

    # value 2: activations staged with cp.async instead of TMA, value 4: register epilogue instead of the staged one
    capi.lib().pwgb_debug_set(1, int(os.environ["PWGB_TC_VARIANT"]))
for spec in sys.argv[1:]:
    c, k, d, T, B = [int(v) for v in spec.split(",")]
    x = torch.randn(B, c, T, device=dev)
    w = torch.randn(c, c, k, device=dev) / (c * k) ** 0.5
    b = torch.randn(c, device=dev)
    res = torch.randn(B, c, T, device=dev)
    for _ in range(3):
        y = ops.conv1d(x, w, b, padding=(k - 1) // 2 * d, dilation=d, pre_slope=0.1, residual=res)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        y = ops.conv1d(x, w, b, padding=(k - 1) // 2 * d, dilation=d, pre_slope=0.1, residual=res)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    fl = 2.0 * B * T * c * c * k
    by = 4.0 * 3 * B * c * T
    print(f"conv c{c} k{k} d{d} T{T} B{B}: {ms:.3f} ms  {fl/ms/1e9:.1f} TFLOP/s(alg)  {by/ms/1e6:.0f} GB/s(alg)")
