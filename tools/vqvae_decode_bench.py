"""Conversion throughput of a corpus of unequal utterances with the VQ-VAE (vctk ``lg`` shape: local and global
conditioning), three ways.

    python tools/vqvae_decode_bench.py [--utts 64] [--min-frames 40] [--max-frames 400] [--rounds 3] [--out FILE]

Workload: ``VQVAE`` of the vctk_lg fixture's configuration with synthetic weights, ``--utts`` waveforms whose lengths
are seeded uniform in [min, max] frames times the hop plus a seeded remainder (a real test set has almost no two equal
lengths), each with its local track and a speaker id.  Each round converts the whole set once per mode, in alternating
order, to PCM16 and indices on the host: batch 1 (``encode`` + ``decode`` per utterance, the reference's loop, eager),
``Decoder(exact=True)`` (batches of equal lengths) and ``Decoder(ragged=True)`` (any lengths, per-item masks); the time
is wall clock to the last synchronise.  One untimed pass per mode first captures its graphs.  The card's name and power
limit are printed with the numbers: they are part of them."""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ragged_decode_bench import _card  # noqa: E402

LG = {"in_channels": 1, "out_channels": 1, "num_embeds": 512, "embed_dim": 256, "num_global_embeds": 128,
      "global_embed_dim": 128, "num_local_embeds": 2, "local_embed_dim": 32,
      "encoder_conf": {"out_channels": 256, "downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 1024},
      "decoder_conf": {"in_channels": 416, "upsample_scales": [4, 4, 2, 2], "channels": 512, "stacks": 3}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--min-frames", type=int, default=40)
    ap.add_argument("--max-frames", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vqvae_decode_bench: needs a CUDA device (no CPU timing)")
    import __graft_entry__

    __graft_entry__.build()
    from oracle import synth
    from parallelwavegan_b200 import decode, models

    dev = torch.device("cuda:0")
    m = models.VQVAE(**copy.deepcopy(LG))
    spec = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(synth.synth_state_dict(spec, 11, 1.0))
    m.remove_weight_norm()
    m = m.to(dev).eval()
    hop = m.hop
    rng = np.random.default_rng(a.seed)
    lens = [int(f) * hop + int(r) for f, r in zip(rng.integers(a.min_frames, a.max_frames + 1, a.utts), rng.integers(0, hop, a.utts))]
    waves = [(0.3 * rng.standard_normal(L)).astype(np.float32) for L in lens]
    locs = [rng.standard_normal((-(-L // hop), 2)).astype(np.float32) for L in lens]
    spk = [int(v) for v in rng.integers(0, 128, a.utts)]

    @torch.no_grad()
    def batch1():
        out = {}
        for i, w in enumerate(waves):
            x = torch.from_numpy(w).pin_memory().to(dev, non_blocking=True).reshape(1, 1, -1)
            l = torch.from_numpy(locs[i].T.copy()).to(dev)[None]
            idx = m.encode(x)
            y = m.decode(idx, l, torch.tensor([spk[i]], device=dev))
            out[i] = (decode.pcm16(y[0, 0]).cpu().numpy(), idx[0].cpu().numpy())
        return out

    decs = {"exact": decode.Decoder(m, exact=True, max_batch=a.max_batch),
            "ragged": decode.Decoder(m, ragged=True, max_batch=a.max_batch)}
    modes = {"batch1": batch1, **{k: (lambda d=d: d.convert(waves, locs, spk)) for k, d in decs.items()}}
    results = {}
    for k, fn in modes.items():  # graphs and caches
        results[k] = fn()
    torch.cuda.synchronize()
    same = {k: sum(np.array_equal(results[k][i][1], results["batch1"][i][1]) for i in range(a.utts)) for k in results}
    times = {k: [] for k in modes}
    for r in range(a.rounds):
        order = list(modes) if r % 2 == 0 else list(reversed(modes))
        for k in order:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            modes[k]()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    name, pl = _card()
    res = {"card": name, "power_limit": pl, "utts": a.utts, "samples": sum(lens), "max_batch": a.max_batch,
           "rounds": a.rounds, "indices_equal_to_batch1": same}
    for k, ts in times.items():
        best = min(ts)
        res[k] = {"wall_s": [round(t, 4) for t in ts], "utts_per_s_best": round(a.utts / best, 1)}
    res["ragged_over_batch1"] = round(min(times["batch1"]) / min(times["ragged"]), 2)
    res["ragged_over_exact"] = round(min(times["exact"]) / min(times["ragged"]), 2)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
