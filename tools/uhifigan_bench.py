#!/usr/bin/env python
"""UHiFiGAN measurements on one GPU; prints one JSON line.

* inference of the opencpop recipe's generator (egs/opencpop/voc1/conf/uhifigan.v1.yaml, weight norm removed, eval
  mode) on a batch of 16 x 400 frames (hop 300): ms per forward from device events with the L2 flushed (256 MiB
  write) before each step, samples/s, libpwgb launches per forward, and rel-L2 of utterance 0 against the CPU oracle;
* the decoder's four skip-concatenation conv-transposes at that batch: the two-source entry against torch.cat + the
  single-source entry, alternated step by step in the same run;
* the card's name and power limit, read in the same call.

    python tools/uhifigan_bench.py [--steps 10] [--warmup 3] [--batch 16] [--frames 400]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

OPENCPOP = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[5, 5, 4, 3],
                downsample_kernel_sizes=[10, 10, 8, 6], upsample_scales=[3, 4, 5, 5], upsample_kernel_sizes=[6, 8, 10, 10],
                resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], dropout=0.1,
                use_additional_convs=True, bias=True, nonlinear_activation="LeakyReLU",
                nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [f.strip() for f in out.split(",")[:2]]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # the measurement stands without it, but says so
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({type(e).__name__})"}


def timed(fns, steps, warmup, flush):
    """Mean device time (ms) of each callable, alternated step by step, L2 flushed before every call."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    evs = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)] for _ in fns]
    for i in range(steps):
        for fn, ev in zip(fns, evs):
            flush.zero_()
            ev[i][0].record()
            fn()
            ev[i][1].record()
    torch.cuda.synchronize()
    return [sum(a.elapsed_time(b) for a, b in ev) / steps for ev in evs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=400)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("uhifigan_bench: needs a CUDA device (no CPU measurement)")
    import __graft_entry__

    __graft_entry__.build()
    from oracle import synth
    from oracle.ref_ops import fold_weight_norm
    from oracle.ref_uhifigan import uhifigan_generator
    from parallelwavegan_b200 import capi, models, ops

    dev = torch.device("cuda:0")
    B, F, hop = args.batch, args.frames, 300
    m = models.UHiFiGANGenerator(**OPENCPOP)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 91, 1.0)
    m.load_state_dict(sd)
    m.remove_weight_norm()
    m = m.to(dev).eval()
    c = synth.randn((B, 80, F), 92).to(dev)
    e = synth.randn((B, 1, F * hop), 93, 0.3).to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    with torch.no_grad():
        y = m(c, None, e)
        torch.cuda.synchronize()
        capi.reset_launch_count()
        m(c, None, e)
        torch.cuda.synchronize()
        launches = capi.launch_count()
        (ms,) = timed([lambda: m(c, None, e)], args.steps, args.warmup, flush)
    ref = uhifigan_generator(fold_weight_norm(sd), e[:1].cpu(), c[:1].cpu(), OPENCPOP)
    rel = float((y[:1].cpu().double() - ref.double()).norm() / ref.double().norm())

    # the decoder's conv-transposes at this batch: inputs of the shapes the model feeds them
    concat = []
    t, ch = F, 32 * 16
    with torch.no_grad():
        for i, s in enumerate(OPENCPOP["upsample_scales"]):
            x1 = torch.randn(B, ch, t, device=dev)
            x2 = torch.randn(B, ch, t, device=dev)
            w = torch.randn(2 * ch, ch // 2, 2 * s, device=dev) / (2 * ch) ** 0.5
            b = torch.randn(ch // 2, device=dev)
            kw = dict(stride=s, padding=s // 2 + s % 2, output_padding=s % 2, pre_slope=0.1)
            two = lambda: ops.conv_transpose1d_cat_raw(x1, x2, w, b, **kw)  # noqa: E731
            one = lambda: ops.conv_transpose1d_raw(torch.cat((x1, x2), dim=1), w, b, **kw)  # noqa: E731
            same = torch.equal(two(), one())
            ms_two, ms_one = timed([two, one], args.steps, args.warmup, flush)
            concat.append({"shape": f"{ch}+{ch}->{ch // 2} s{s}", "t_in": t, "two_source_ms": round(ms_two, 4),
                           "cat_plus_single_ms": round(ms_one, 4), "bit_identical": same})
            t, ch = t * s, ch // 2
    line = {
        "workload": f"UHiFiGAN opencpop inference, batch {B} x {F} frames (hop {hop}), eval, weight norm removed",
        "ms_per_step": round(ms, 3),
        "samples_per_s": round(B * F * hop / (ms / 1e3)),
        "launches_per_step": launches,
        "rel_l2_utt0_vs_oracle": rel,
        "concat_conv_transpose": concat,
        "timing": f"device events, mean of {args.steps} steps after {args.warmup} warm-up, L2 flushed (256 MiB write) before each",
        "gpu": card(),
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
