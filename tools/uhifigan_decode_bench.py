"""SineGen kernel time and U-Net HiFi-GAN decode throughput.

    python tools/uhifigan_decode_bench.py [--utts 64] [--min-frames 100] [--max-frames 800] [--rounds 3] [--out FILE]

SineGen: ``ops.sine_gen`` (pwgb_sine_gen_forward, five launches) on log-f0 contours as the dumps hold them, with the
draws made beforehand, timed with CUDA events at the bench.py shape of the opencpop recipe (16 rows of 400 frames x hop
300 = 120000 samples) and on one 10-minute row at 24 kHz (14.4 M samples).  Bytes are counted from the shapes: f0 and
the noise draw read once, sine_waves, uv and noise written once (20 bytes per sample at harmonic_num 0).  The kernel
reads f0 three times (once per chunk pass) and moves 16 bytes per 2048-sample chunk and scan, so the traffic it issues
is 28 bytes per sample; the rate below counts 20.

Decoder: the opencpop U-Net HiFi-GAN (weight norm removed, synthetic weights), ``--utts`` utterances of seeded frame
counts in [min, max] with their excitations from ``features.excitation`` (made beforehand), decoded to PCM16 on the host
by ``Decoder(exact=True)`` (equal lengths), ``Decoder(exact=False)`` (zero-padded buckets of 32 frames) and a loop of
``inference`` + PCM16 + copy per utterance, in alternating order; wall clock to the last synchronise, after one
untimed pass per mode.  The card's name and power limit are printed with the numbers: they are part of them."""
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

OPENCPOP = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[5, 5, 4, 3],
                downsample_kernel_sizes=[10, 10, 8, 6], upsample_scales=[3, 4, 5, 5], upsample_kernel_sizes=[6, 8, 10, 10],
                resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], dropout=0.1)
SR, HOP = 24000, 300
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


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


def sine_kernel(dev, B, T, reps, seed):
    from oracle import ref_sine
    from parallelwavegan_b200 import ops

    f0 = torch.from_numpy(np.stack([ref_sine.f0_contour(T, seed + b, log=True) for b in range(B)])).to(dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    rand_ini = torch.rand(B, 1, device=dev, generator=g)
    n = torch.randn(B, T, 1, device=dev, generator=g)

    def run():
        return ops.sine_gen(f0, 0, SR, 0.1, 0.003, 0, rand_ini, n)

    run()
    ms = [_events_ms(run, reps) for _ in range(5)]
    t = float(np.median(ms))
    nbytes = 20 * B * T
    return {"B": B, "T": T, "ms": ms, "median_ms": t, "bytes": nbytes, "GB_per_s": nbytes / t / 1e6,
            "share_of_hbm": nbytes / (t * 1e-3) / HBM_BYTES_PER_S}


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
        raise SystemExit("uhifigan_decode_bench: needs a CUDA device (no CPU numbers)")
    import __graft_entry__

    __graft_entry__.build()
    from oracle import ref_sine, synth
    from parallelwavegan_b200 import decode, features, models

    dev = torch.device("cuda:0")
    res = {"card": None, "power_limit": None}
    res["sine_gen"] = {"16x400x300": sine_kernel(dev, 16, 400 * HOP, 50, 1), "10min_row": sine_kernel(dev, 1, 600 * SR, 10, 2)}

    m = models.UHiFiGANGenerator(**OPENCPOP)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 11, 1.15))
    m.remove_weight_norm()
    m = m.to(dev).eval()
    rng = np.random.default_rng(a.seed)
    lens = rng.integers(a.min_frames, a.max_frames + 1, a.utts)
    mels = [rng.standard_normal((int(L), 80)).astype(np.float32) for L in lens]
    gen = torch.Generator(device=dev).manual_seed(a.seed)
    excs = [features.excitation(torch.from_numpy(ref_sine.f0_contour(int(L), 100 + i, low=120.0, high=700.0, log=True)).to(dev),
                                int(L), SR, HOP, generator=gen).cpu().numpy() for i, L in enumerate(lens)]
    decs = {"exact": decode.Decoder(m, use_graphs=True, max_batch=16, exact=True),
            "bucketed": decode.Decoder(m, use_graphs=True, max_batch=16, exact=False, bucket_frames=32)}

    def per_utterance():
        out = {}
        with torch.no_grad():
            for i, (c, e) in enumerate(zip(mels, excs)):
                y = m.inference(e, c=c)
                out[i] = decode.pcm16(y[:, 0].contiguous()).cpu().numpy()
        return out

    modes = {"exact": lambda: decs["exact"].decode(mels, excitations=excs),
             "bucketed": lambda: decs["bucketed"].decode(mels, excitations=excs), "inference_loop": per_utterance}
    for f in modes.values():
        f()
    times = {k: [] for k in modes}
    order = list(modes)
    for r in range(a.rounds):
        for k in (order if r % 2 == 0 else order[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            modes[k]()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    res.update({"utts": a.utts, "frames": [int(lens.min()), int(lens.max()), int(lens.sum())], "decode_s": times,
                "utts_per_s": {k: a.utts / float(np.median(v)) for k, v in times.items()}})
    res["card"], res["power_limit"] = _card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
