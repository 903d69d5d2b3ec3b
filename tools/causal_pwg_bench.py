"""PWG v1 generator forward, centred vs causal (use_causal_conv=True), timed alternately in one process: B x 25600
samples, L2 flushed before every call, CUDA events, median of the repeats.  The causal layer moves the same bytes and
does the same MACs as the centred one (only the tap origin of the activation windows moves), so the two should time
within noise.  Prints the card name and power limit, and checks both outputs against the CPU oracle at B = 1.

    python tools/causal_pwg_bench.py [B ...]        # default: 1 16"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import ref_causal_pwg, ref_ops  # noqa: E402
from parallelwavegan_b200 import models  # noqa: E402
from parallelwavegan_b200 import synth_weights as synth  # noqa: E402

T = 25600
REPEATS = 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def build(causal, dev):
    m = models.ParallelWaveGANGenerator(use_causal_conv=causal)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.0)
    m.load_state_dict(sd)
    m.remove_weight_norm()
    return m.eval().to(dev), {k: v.detach().cpu() for k, v in m.state_dict().items()}


def main():
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    arms = {"centred": build(False, dev), "causal": build(True, dev)}
    out = {"card": card(), "T": T}
    with torch.no_grad():
        for B in [int(a) for a in (sys.argv[1:] or ["1", "16"])]:
            g = torch.Generator().manual_seed(B)
            z = torch.randn(B, 1, T, generator=g).to(dev)
            c = torch.randn(B, 80, T // 256 + 4, generator=g).to(dev)
            for m, _ in arms.values():
                for _ in range(3):
                    m(z, c)
            torch.cuda.synchronize()
            ts = {k: [] for k in arms}
            for _ in range(REPEATS):
                for k, (m, _) in arms.items():
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    m(z, c)
                    e1.record()
                    torch.cuda.synchronize()
                    ts[k].append(e0.elapsed_time(e1))
            row = {k: {"ms_median": sorted(v)[REPEATS // 2], "ms_min": min(v), "ms_max": max(v)} for k, v in ts.items()}
            row["causal_over_centred"] = row["causal"]["ms_median"] / row["centred"]["ms_median"]
            if B == 1:
                for k, (m, w) in arms.items():
                    cfg = dict(ref_ops.PWG_V1, use_causal_conv=k == "causal")
                    ref = ref_causal_pwg.pwg_generator(w, z.cpu(), c.cpu(), cfg)
                    y = m(z, c).cpu()
                    err = float((y.double() - ref.double()).norm() / ref.double().norm())
                    row[k]["rel_l2_vs_oracle"] = err
                    assert err < 1e-3, (k, err)
            out[f"B{B}"] = row
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
