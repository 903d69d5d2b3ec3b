"""Per-push latency of streaming the causal HiFi-GAN v1 generator (parallelwavegan_b200.streaming.CausalHiFiGANStream)
with synthetic weights, for batch sizes B, chunks of 1, 4, 16 and 64 frames (hop 256), CUDA graphs on and off.

Each configuration streams a 256-frame utterance (65536 samples per item) PASSES times.  A push is timed with CUDA
events recorded around it and a synchronise after it, so a latency includes the host's launch work whenever the GPU
waits for it.  Reported: median / min / max push latency, the streamed real-time factor (GPU time of all pushes over
the audio's duration at 22050 Hz: below 1 is faster than real time), the libpwgb kernel launches of one steady-state
eager push (convs, conv-transpose weight preparation and carries; the few torch copies are not counted), and the
whole-utterance forward of the same audio (B x 65536 samples, one call) for comparison.  Every timed stream is checked against
``model.inference`` of each item in the same run: the per-item inference's 32 -> 1 output conv has 65536 output samples
and takes conv1d_fewcout_long_kernel, which sums in another order than the generic kernel every stream conv takes, so
the check is rel-L2 <= 1e-6 (bit identity holds up to 15 frames, tests/test_gpu_hifigan_stream.py).  Prints the card
name and power limit of the same run, as one JSON document.

    python tools/hifigan_stream_bench.py [B ...]        # default: 1 16"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from parallelwavegan_b200 import capi, models  # noqa: E402
from parallelwavegan_b200 import synth_weights as synth  # noqa: E402
from parallelwavegan_b200.streaming import CausalHiFiGANStream  # noqa: E402

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
    m = models.HiFiGANGenerator(use_causal_conv=True)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.15))
    m.remove_weight_norm()
    m = m.eval().to(dev)
    hop = 256
    out = {"card": card(), "frames": FRAMES, "samples_per_item": FRAMES * hop, "sample_rate_for_rtf": SR}
    with torch.no_grad():
        for B in [int(a) for a in (sys.argv[1:] or ["1", "16"])]:
            g = torch.Generator().manual_seed(B)
            c = torch.randn(B, FRAMES, 80, generator=g).to(dev)
            ref = torch.stack([m.inference(c[b]).t() for b in range(B)])
            cw = c.transpose(1, 2).contiguous()
            for _ in range(3):
                m(cw)
            ts = []
            for _ in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                m(cw)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            row = {"whole_utterance_forward": stats(ts)}
            audio_s = FRAMES * hop / SR
            for graphs in (False, True):
                for n in CHUNKS:
                    st = CausalHiFiGANStream(m, batch=B, use_graphs=graphs)
                    st.push(c[:, :n])  # warm-up: caches, weight packing, graph capture
                    capi.reset_launch_count()
                    st.push(c[:, n:2 * n])
                    launches = capi.launch_count()  # a steady-state push (0 with graphs: the replay launches nothing)
                    lat, ys = [], []
                    for _ in range(PASSES):
                        st.reset()
                        ys.clear()
                        for j in range(0, FRAMES, n):
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            y = st.push(c[:, j:j + n])
                            e1.record()
                            torch.cuda.synchronize()
                            lat.append(e0.elapsed_time(e1))
                            ys.append(y)
                    y = torch.cat(ys, -1)
                    s = stats(lat)
                    s["rtf"] = sum(lat) / PASSES / 1e3 / audio_s
                    if not graphs:
                        s["libpwgb_launches_per_push"] = launches
                    s["bit_identical_to_inference"] = torch.equal(y, ref)
                    s["rel_l2_vs_inference"] = float((y - ref).double().norm() / ref.double().norm())
                    row[f"{'graph' if graphs else 'eager'}_chunk{n}"] = s
                    assert s["rel_l2_vs_inference"] <= 1e-6, (B, graphs, n, s["rel_l2_vs_inference"])
            out[f"B{B}"] = row
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
