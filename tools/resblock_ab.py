"""A/B timing of the fused ResBlock pair kernels at the 18 HiFi-GAN v1 pair shapes of the bench forward (B = 16):
the conv-split kernel against the lockstep one (pwgb_debug_set(3, 1)), alternating in one process, CUDA events around
`--reps` launches per sample.  Checks that both give the same bits, and prints each pair's time against its floors:
algorithmic bytes over 3.35 TB/s and the bf16x3 MMAs of both convs at 989 TFLOP/s (H100 SXM data-sheet figures for a
700 W card)."""
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
    args = ap.parse_args()
    __graft_entry__.build()
    from parallelwavegan_b200 import capi, ops

    lib = capi.lib()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu:", q)
    cases = [(C, k, d) for C in (64, 32) for k in (3, 7, 11) for d in (1, 3, 5)]
    print(f"{'C':>3s} {'k':>3s} {'d':>3s} {'split ms':>18s} {'lockstep ms':>18s} {'ratio':>6s} {'bytes fl':>9s} {'MMA fl':>8s}"
          f"  x floor  plan split / lockstep")
    tot_s = tot_l = 0.0
    for C, k, d in cases:
        B, T = 16, 51200 if C == 64 else 102400
        acc = d == 5 and k > 3  # the MRF-summing last pair of the k = 7 and 11 blocks
        g = torch.Generator(device=dev).manual_seed(C + k + d)
        x = torch.randn(B, C, T, device=dev, generator=g)
        w1 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
        w2 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
        b1 = 0.1 * torch.randn(C, device=dev, generator=g)
        b2 = 0.1 * torch.randn(C, device=dev, generator=g)
        out = torch.zeros_like(x)
        plans = []

        def run(lockstep, n):
            lib.pwgb_debug_set(3, int(lockstep))
            for _ in range(n):
                ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=SLOPE, out=out, accumulate=acc,
                                  out_scale=1.0 / 3.0)

        with torch.no_grad():
            ys = []
            for lockstep in (False, True):
                lib.pwgb_debug_set(3, int(lockstep))
                pl = ops.resblock_pair_plan(C, T, k, d, batch=B)
                plans.append(f"{pl['variant']} na{pl['na']} nb{pl['nb']} ns{pl['ns']}")
                out.zero_()
                run(lockstep, 1)
                ys.append(out.clone())
            assert torch.equal(ys[0], ys[1]), (C, k, d)
            times = {False: [], True: []}
            for _ in range(args.rounds):
                for lockstep in (False, True):
                    run(lockstep, 2)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run(lockstep, args.reps)
                    e1.record()
                    torch.cuda.synchronize()
                    times[lockstep].append(e0.elapsed_time(e1) / args.reps)
        lib.pwgb_debug_set(3, 0)
        ts, tl = times[False], times[True]
        bytes_floor = 4.0 * B * C * T * (2 + acc) / 3.35e12 * 1e3
        mma_floor = 3 * 2 * 2.0 * B * C * T * C * k / 989e12 * 1e3
        tot_s += min(ts)
        tot_l += min(tl)
        print(f"{C:3d} {k:3d} {d:3d} {min(ts):8.3f}-{max(ts):8.3f} {min(tl):8.3f}-{max(tl):8.3f} {min(ts) / min(tl):6.3f} "
              f"{bytes_floor:9.3f} {mma_floor:8.3f} {min(ts) / max(bytes_floor, mma_floor):7.2f}  {plans[0]} / {plans[1]}")
    print(f"sum of the 18 pairs (best sample): split {tot_s:.3f} ms, lockstep {tot_l:.3f} ms, ratio {tot_s / tot_l:.3f}")
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw,clocks_throttle_reasons.active", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("gpu after:", q)


if __name__ == "__main__":
    main()
