"""Decode throughput of a corpus of unequal utterances with HiFi-GAN v1, per Decoder mode, and the cost of the length
mask in the fused ResBlock pairs.

    python tools/ragged_decode_bench.py [--utts 64] [--min-frames 100] [--max-frames 800] [--rounds 3] [--out FILE]

Workload: HiFi-GAN v1 (weight norm removed, synthetic weights), ``--utts`` utterances whose frame counts are seeded
uniform in [min, max] (a real test set has almost no two equal lengths).  Each round decodes the whole set once per mode,
``exact=True`` (batches of equal lengths), ``ragged=True`` (any lengths, length mask) and ``exact=False`` (zero-padded
length buckets), in alternating order, to PCM16 on the host; the time is wall clock to the decoder's last synchronise.
One untimed pass per mode first captures its graphs.  Then the 36 ResBlock pairs of v1 at the bench.py shape (16
utterances of 400 frames, every item full length) are timed with CUDA events, masked and unmasked alternated, and so is
the whole generator forward with and without ``lengths``.  The card's name and power limit are printed with the
numbers: they are part of them."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

V1 = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 8, 2, 2],
          upsample_kernel_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3)


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:  # no nvidia-smi: the number goes out without its power limit, and says so
        pl = "unknown"
    return name, pl


def _events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--min-frames", type=int, default=100)
    ap.add_argument("--max-frames", type=int, default=800)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_decode_bench: needs a CUDA device (no CPU numbers)")
    import __graft_entry__

    __graft_entry__.build()
    from oracle import synth
    from parallelwavegan_b200 import decode, models, ops

    dev = torch.device("cuda:0")
    m = models.HiFiGANGenerator(**V1)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 7, 1.15))
    m.remove_weight_norm()
    m = m.to(dev).eval()
    rng = np.random.default_rng(a.seed)
    lens = rng.integers(a.min_frames, a.max_frames + 1, a.utts)
    mels = [rng.standard_normal((int(L), 80)).astype(np.float32) for L in lens]
    modes = {"exact": dict(exact=True), "ragged": dict(ragged=True), "bucketed": dict(exact=False)}
    decs = {k: decode.Decoder(m, use_graphs=True, max_batch=16, bucket_frames=32, **kw) for k, kw in modes.items()}
    for d in decs.values():
        d.decode(mels)
    times = {k: [] for k in modes}
    order = list(modes)
    for r in range(a.rounds):
        for k in (order if r % 2 == 0 else order[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            decs[k].decode(mels)
            times[k].append(time.perf_counter() - t0)
    res = {"card": None, "power_limit": None, "utts": a.utts, "frames": [int(lens.min()), int(lens.max()), int(lens.sum())],
           "decode_s": {k: v for k, v in times.items()},
           "utts_per_s": {k: a.utts / float(np.median(v)) for k, v in times.items()}}

    # the mask's cost at the bench.py shape: every item full length
    B, T = 16, 400
    lengths = torch.full((B,), T, dtype=torch.int32, device=dev)
    zero = torch.zeros_like(lengths)
    g = torch.Generator().manual_seed(1)
    pair_ms = {"unmasked": 0.0, "masked": 0.0}
    rate = 1
    for i, s in enumerate(V1["upsample_scales"]):
        rate *= s
        C = 256 >> i
        x = torch.randn(B, C, T * rate, generator=g).to(dev)
        out = torch.empty_like(x)
        mask = (zero, lengths, rate, 0)
        for k in V1["resblock_kernel_sizes"]:
            w1 = (torch.randn(C, C, k, generator=g) * 0.05).to(dev)
            w2 = (torch.randn(C, C, k, generator=g) * 0.05).to(dev)
            b1 = torch.randn(C, generator=g).to(dev) * 0.1
            b2 = torch.randn(C, generator=g).to(dev) * 0.1
            for dl in (1, 3, 5):
                def run(mk):
                    return lambda: ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=dl, slope=0.1, out=out, mask=mk)
                for f in (run(None), run(mask)):
                    f()
                for rep in range(3):
                    for name, mk in (("unmasked", None), ("masked", mask)) if rep % 2 == 0 else (("masked", mask), ("unmasked", None)):
                        pair_ms[name] += _events_ms(run(mk), 10) / 3
    res["pairs_ms_36"] = pair_ms
    c = torch.randn(B, 80, T, generator=g).to(dev)
    fwd = {"forward": lambda: m(c), "forward_lengths": lambda: m(c, lengths)}
    with torch.no_grad():
        for f in fwd.values():
            f()
        fw = {k: [] for k in fwd}
        for rep in range(6):
            for k in (list(fwd) if rep % 2 == 0 else list(fwd)[::-1]):
                fw[k].append(_events_ms(fwd[k], 5))
    res["forward_ms"] = {k: float(np.median(v)) for k, v in fw.items()}
    res["card"], res["power_limit"] = _card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
