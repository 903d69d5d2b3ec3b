"""Per-push latency of streaming the causal MelGAN v1 (512 channels, scales [8, 8, 2, 2], 3 stacks) and the causal
multi-band MelGAN v2 (384 channels, scales [8, 4, 2], 4 stacks, 4-band PQMF) generators
(parallelwavegan_b200.streaming.CausalMelGANStream), synthetic weights with weight norm removed, for batch sizes B,
chunks of 1, 4, 16 and 64 frames after a min_first_frames opening push, CUDA graphs on and off.

Each configuration streams a 263-frame utterance (the 7-frame opening push, then 256 frames; 256 output samples per
frame for both models) PASSES times, and flushes.  A push is timed with CUDA events recorded around it and a
synchronise after it, so a latency includes the host's launch work whenever the GPU waits for it.  Reported: median /
min / max latency of the chunk pushes, the streamed real-time factor (GPU time of all pushes and the flush over the
audio's duration at 22050 Hz: below 1 is faster than real time), the libpwgb kernel launches of one steady-state eager
push (the few torch copies are not counted), and the whole-utterance forward of the same audio (``inference``'s forward
and PQMF synthesis on the B utterances, one call) for comparison.  Every timed stream is checked against
``model.inference`` of each item in the same run, after the PQMF delay: the per-item inference's output conv has 67328
output samples and takes conv1d_fewcout_long_kernel, which sums in another order than the generic kernel every stream
conv takes, so the check is rel-L2 <= 1e-6 (bit identity holds below 4096 output-conv samples,
tests/test_gpu_melgan_stream.py).  Prints the card name and power limit of the same run, as one JSON document.

    python tools/melgan_stream_bench.py [B ...]        # default: 1 16"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from parallelwavegan_b200 import capi, models  # noqa: E402
from parallelwavegan_b200 import synth_weights as synth  # noqa: E402
from parallelwavegan_b200.layers import PQMF  # noqa: E402
from parallelwavegan_b200.streaming import CausalMelGANStream  # noqa: E402

MODELS = {
    "melgan_v1": dict(in_channels=80, out_channels=1, kernel_size=7, channels=512, upsample_scales=[8, 8, 2, 2], stacks=3,
                      use_causal_conv=True),
    "mb_melgan_v2": dict(in_channels=80, out_channels=4, kernel_size=7, channels=384, upsample_scales=[8, 4, 2], stacks=4,
                         use_causal_conv=True),
}
OPEN = 7
FRAMES = OPEN + 256
CHUNKS = (1, 4, 16, 64)
PASSES = 2
SR = 22050


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def stats(v):
    v = sorted(v)
    return {"ms_median": v[len(v) // 2], "ms_min": v[0], "ms_max": v[-1], "pushes": len(v)}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    y = fn()
    e1.record()
    torch.cuda.synchronize()
    return y, e0.elapsed_time(e1)


def build(name, dev):
    kw = MODELS[name]
    m = models.MelGANGenerator(**kw)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.0))
    m.remove_weight_norm()
    m = m.eval().to(dev)
    if kw["out_channels"] > 1:
        m.pqmf = PQMF(kw["out_channels"]).to(dev)
    return m


def bench_model(name, Bs, dev):
    m = build(name, dev)
    res = {}
    for B in Bs:
        g = torch.Generator().manual_seed(B)
        c = torch.randn(B, FRAMES, 80, generator=g).to(dev)
        probe = CausalMelGANStream(m, batch=B, use_graphs=False)
        assert probe.min_first_frames == OPEN, probe.min_first_frames
        delay = probe.delay
        ref = F.pad(torch.stack([m.inference(c[b]).t() for b in range(B)]), (delay, 0))
        samples = ref.shape[-1] - delay
        cw = c.transpose(1, 2).contiguous()

        def whole():
            y = m(cw)
            return m.pqmf.synthesis(y) if m.pqmf is not None else y

        for _ in range(3):
            whole()
        row = {"samples_per_item": samples, "delay_samples": delay,
               "whole_utterance_forward": stats([timed(whole)[1] for _ in range(5)])}
        audio_s = samples / SR
        for graphs in (False, True):
            for n in CHUNKS:
                st = CausalMelGANStream(m, batch=B, use_graphs=graphs)
                st.push(c[:, :OPEN])  # warm-up: caches, weight packing, graph capture of both lengths
                st.push(c[:, OPEN:OPEN + n])
                capi.reset_launch_count()
                st.push(c[:, OPEN + n:OPEN + 2 * n])
                launches = capi.launch_count()  # a steady-state push (0 with graphs: the replay launches nothing)
                lat, total = [], 0.0
                for _ in range(PASSES):
                    st.reset()
                    y, t = timed(lambda: st.push(c[:, :OPEN]))
                    ys = [y]
                    total += t
                    for j in range(OPEN, FRAMES, n):
                        y, t = timed(lambda: st.push(c[:, j:j + n]))
                        lat.append(t)
                        total += t
                        ys.append(y)
                    y, t = timed(st.flush)
                    total += t
                    ys.append(y)
                y = torch.cat(ys, -1)
                s = stats(lat)
                s["rtf"] = total / PASSES / 1e3 / audio_s
                if not graphs:
                    s["libpwgb_launches_per_push"] = launches
                s["bit_identical_to_inference"] = torch.equal(y, ref)
                s["rel_l2_vs_inference"] = float((y - ref).double().norm() / ref.double().norm())
                row[f"{'graph' if graphs else 'eager'}_chunk{n}"] = s
                assert s["rel_l2_vs_inference"] <= 1e-6, (name, B, graphs, n, s["rel_l2_vs_inference"])
        res[f"B{B}"] = row
    return res


def main():
    dev = torch.device("cuda:0")
    Bs = [int(a) for a in (sys.argv[1:] or ["1", "16"])]
    out = {"card": card(), "frames": FRAMES, "opening_push_frames": OPEN, "sample_rate_for_rtf": SR}
    with torch.no_grad():
        for name in MODELS:
            out[name] = bench_model(name, Bs, dev)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
