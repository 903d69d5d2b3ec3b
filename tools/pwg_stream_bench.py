"""Per-push latency of streaming the causal PWG v1 generator (parallelwavegan_b200.streaming.CausalPWGStream) with
synthetic weights, for batch sizes B, chunks of 1, 4, 16 and 64 frames (hop 256), CUDA graphs on and off.

Each configuration streams a 256-frame utterance (65536 samples per item) PASSES times.  A push is timed with CUDA
events recorded around it and a synchronise after it, so a latency includes the host's launch work whenever the GPU
waits for it.  Reported: median / min / max push latency, the streamed real-time factor (GPU time of all pushes over
the audio's duration at 22050 Hz: below 1 is faster than real time), and the whole-utterance forward of the same audio
(B x 65536 samples, one call) for comparison.  Every timed stream is checked against ``model.inference`` of each item:
bit for bit while a push has at most 65536 samples in all (B x chunk x 256), so that its 64 -> 1 output conv takes
conv1d_small_cout_kernel as the per-item inference does; above that the push's output conv takes
conv1d_fewcout_long_kernel, which sums in another order, and the check is rel-L2 <= 1e-6.  Prints the card name and
power limit of the same run, as one JSON document.

    python tools/pwg_stream_bench.py [B ...]        # default: 1 16"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from parallelwavegan_b200 import models  # noqa: E402
from parallelwavegan_b200 import synth_weights as synth  # noqa: E402
from parallelwavegan_b200.streaming import CausalPWGStream  # noqa: E402

FRAMES = 256
CHUNKS = (1, 4, 16, 64)
PASSES = 2
SR = 22050


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def stats(v):
    v = sorted(v)
    return {"ms_median": v[len(v) // 2], "ms_min": v[0], "ms_max": v[-1], "pushes": len(v)}


def main():
    dev = torch.device("cuda:0")
    m = models.ParallelWaveGANGenerator(use_causal_conv=True)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.0))
    m.remove_weight_norm()
    m = m.eval().to(dev)
    hop = m.upsample_factor
    out = {"card": card(), "frames": FRAMES, "samples_per_item": FRAMES * hop, "sample_rate_for_rtf": SR}
    with torch.no_grad():
        for B in [int(a) for a in (sys.argv[1:] or ["1", "16"])]:
            g = torch.Generator().manual_seed(B)
            c = torch.randn(B, FRAMES, 80, generator=g).to(dev)
            z = torch.randn(B, 1, FRAMES * hop, generator=g).to(dev)
            ref = torch.stack([m.inference(c=c[b], x=z[b].t()).t() for b in range(B)])
            # whole-utterance forward of the same audio (the inference input: edge-padded by aux_context_window)
            acw = m.aux_context_window
            idx = torch.arange(-acw, FRAMES + acw, device=dev).clamp(0, FRAMES - 1)
            cw = c.transpose(1, 2)[:, :, idx].contiguous()
            for _ in range(3):
                m(z, cw)
            ts = []
            for _ in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                m(z, cw)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            row = {"whole_utterance_forward": stats(ts)}
            audio_s = FRAMES * hop / SR
            for graphs in (False, True):
                for n in CHUNKS:
                    st = CausalPWGStream(m, batch=B, use_graphs=graphs)
                    st.push(c[:, :n], z[:, :, :n * hop])  # warm-up: caches, graph capture
                    lat, ys = [], []
                    for _ in range(PASSES):
                        st.reset()
                        ys.clear()
                        for j in range(0, FRAMES, n):
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            y = st.push(c[:, j:j + n], z[:, :, j * hop:(j + n) * hop])
                            e1.record()
                            torch.cuda.synchronize()
                            lat.append(e0.elapsed_time(e1))
                            ys.append(y)
                    y = torch.cat(ys, -1)
                    s = stats(lat)
                    s["rtf"] = sum(lat) / PASSES / 1e3 / audio_s
                    s["bit_identical_to_inference"] = torch.equal(y, ref)
                    s["rel_l2_vs_inference"] = float((y - ref).double().norm() / ref.double().norm())
                    row[f"{'graph' if graphs else 'eager'}_chunk{n}"] = s
                    if B * n * hop <= 65536:
                        assert s["bit_identical_to_inference"], (B, graphs, n)
                    else:
                        assert s["rel_l2_vs_inference"] <= 1e-6, (B, graphs, n, s["rel_l2_vs_inference"])
            out[f"B{B}"] = row
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
