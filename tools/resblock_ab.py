"""A/B timing of the fused ResBlock pair (ops.resblock_pair, one launch) against the two tensor-core conv launches it
replaces, at the 18 HiFi-GAN v1 pair shapes of the bench forward and at any extra `C,k,d` shapes given (B = 16,
C x T = 64 x 51200), alternating in one process, CUDA events around `--reps` calls per sample.  Checks that both give the
same bits, and prints each pair's times against its floors: algorithmic bytes of the fused pair over 3.35 TB/s and the
bf16x3 MMAs of both convs at 989 TFLOP/s (H100 SXM data-sheet figures for a 700 W card).  A shape the fused kernel has
no plan for is timed as two launches only and printed as "not fused".

    python tools/resblock_ab.py [--reps N] [--rounds N] [C,k,d ...]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import __graft_entry__

SLOPE = 0.1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("shapes", nargs="*", metavar="C,k,d", help="extra pair shapes, timed after the 18 v1 pairs")
    args = ap.parse_args()
    __graft_entry__.build()
    from parallelwavegan_b200 import ops

    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", q)
    v1 = [(C, k, d) for C in (64, 32) for k in (3, 7, 11) for d in (1, 3, 5)]
    extra = [tuple(int(v) for v in s.split(",")) for s in args.shapes]
    print(f"{'C':>3s} {'k':>3s} {'d':>3s} {'fused ms':>17s} {'two launches ms':>17s} {'ratio':>6s} {'bytes fl':>9s} "
          f"{'MMA fl':>8s}  x floor  plan: na, nb, ns")
    tot_f = tot_2 = 0.0
    for C, k, d in v1 + extra:
        B, T = 16, 64 * 51200 // C
        acc = (C, k, d) in v1 and d == 5 and k > 3  # the MRF-summing last pair of the k = 7 and 11 blocks
        g = torch.Generator(device=dev).manual_seed(C + k + d)
        x = torch.randn(B, C, T, device=dev, generator=g)
        w1 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
        w2 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
        b1 = 0.1 * torch.randn(C, device=dev, generator=g)
        b2 = 0.1 * torch.randn(C, device=dev, generator=g)
        out = torch.zeros_like(x)
        plan = ops.resblock_pair_plan(C, T, k, d, batch=B)

        def fused():
            y = ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=SLOPE, out=out, accumulate=acc,
                                  out_scale=1.0 / 3.0)
            assert y is not None, (C, k, d)

        def two_launches():
            xt = ops.conv1d(x, w1, b1, dilation=d, padding=(k - 1) // 2 * d, pre_slope=SLOPE)
            ops.conv1d(xt, w2, b2, padding=(k - 1) // 2, pre_slope=SLOPE, residual=x, out=out, accumulate=acc,
                       out_scale=1.0 / 3.0)

        runs = {"fused": fused, "two": two_launches} if plan else {"two": two_launches}
        with torch.no_grad():
            ys = []
            for fn in runs.values():
                out.zero_()
                fn()
                ys.append(out.clone())
            assert all(torch.equal(ys[0], y) for y in ys), (C, k, d)
            times = {name: [] for name in runs}
            for _ in range(args.rounds):
                for name, fn in runs.items():
                    for _ in range(2):
                        fn()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        fn()
                    e1.record()
                    torch.cuda.synchronize()
                    times[name].append(e0.elapsed_time(e1) / args.reps)
        t2 = times["two"]
        bytes_floor = 4.0 * B * C * T * (2 + acc) / 3.35e12 * 1e3
        mma_floor = 3 * 2 * 2.0 * B * C * T * C * k / 989e12 * 1e3
        if plan:
            tf = times["fused"]
            if (C, k, d) in v1:
                tot_f += min(tf)
                tot_2 += min(t2)
            print(f"{C:3d} {k:3d} {d:3d} {min(tf):8.3f}-{max(tf):8.3f} {min(t2):8.3f}-{max(t2):8.3f} {min(tf) / min(t2):6.3f} "
                  f"{bytes_floor:9.3f} {mma_floor:8.3f} {min(tf) / max(bytes_floor, mma_floor):7.2f}  "
                  f"{plan['na']}, {plan['nb']}, {plan['ns']}")
        else:
            print(f"{C:3d} {k:3d} {d:3d} {'not fused':>17s} {min(t2):8.3f}-{max(t2):8.3f} {'-':>6s} "
                  f"{bytes_floor:9.3f} {mma_floor:8.3f} {'-':>7s}  -")
    print(f"sum of the 18 v1 pairs (best sample): fused {tot_f:.3f} ms, two launches {tot_2:.3f} ms"
          + (f", ratio {tot_f / tot_2:.3f}" if tot_2 else ""))
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw,clocks_throttle_reasons.active", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu after:", q)


if __name__ == "__main__":
    main()
