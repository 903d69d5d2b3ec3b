"""Per-push latency of the causal streams (parallelwavegan_b200.streaming) with synthetic weights, weight norm removed,
for batch sizes B, chunks of 1, 4, 16 and 64 frames, CUDA graphs off and on.  MODEL is

* pwg: the causal PWG v1 generator (CausalPWGStream), hop 256;
* hifigan: the causal HiFi-GAN v1 generator (CausalHiFiGANStream), hop 256;
* hifigan_centred: the centred HiFi-GAN v1 generator (HiFiGANLookaheadStream), hop 256, with its 3258-sample lookahead;
* pwg_centred: the centred PWG v1 generator (PWGLookaheadStream), hop 256, with its 3920-sample lookahead;
* melgan_v1: the causal MelGAN v1 (512 channels, scales [8, 8, 2, 2], 3 stacks; CausalMelGANStream);
* mb_melgan_v2: the causal multi-band MelGAN v2 (384 channels, scales [8, 4, 2], 4 stacks, 4-band PQMF), 256 output
  samples per frame like the others;
* melgan_v1_centred, mb_melgan_v2_centred: the same two models centred (MelGANLookaheadStream), with their 1425- and
  2719-sample lookaheads;
* uhifigan_opencpop_centred: the U-Net HiFi-GAN of the opencpop recipe (UHiFiGANLookaheadStream), hop 300 at 24 kHz,
  excitation pushed with its frames, with its 16231-sample lookahead; 1- and 8-frame chunks;
* vqvae_vctk_lg: the wav2wav conversion of the vctk local- and global-conditioned VQ-VAE recipe (VQVAELookaheadStream),
  hop 64 at 24 kHz, audio and local conditioning pushed together, a target speaker per slot, with its 1305-sample
  lookahead; 1-, 4- and 16-frame chunks;
* dsym_vctk_centred: the discrete-symbol HiFi-GAN of the vctk hubert_voc1 recipe (DiscreteSymbolHiFiGANLookaheadStream),
  HuBERT units and a speaker per slot, hop 320 at 16 kHz, with its 3482-sample lookahead; 1-, 4- and 16-frame chunks;
* dsym_dur_cvss: the duration model of the cvss_c hubert_voc1 recipe (DiscreteSymbolDurationLookaheadStream): 128
  deduplicated units per item (the predictor's bias set so that durations are 0 .. 4 frames), pushed 1, 4 or 16 units
  at a time; a push yields however many frames every slot has queued, so its latency is per push of units and the
  check compares each slot's audio and durations with its own ``synthesis``.

PWG and HiFi-GAN stream a 256-frame utterance (65536 samples per item), the centred ones then flush; the MelGANs
stream a 263-frame one, a 7-frame opening push (their min_first_frames) then 256 frames, and flush; the centred
MelGANs stream 256 frames and flush.  Each configuration streams its utterance PASSES
times.  A push is timed with CUDA events recorded around it and a synchronise after it, so a latency includes the
host's launch work whenever the GPU waits for it.  Reported: median / min / max latency of the chunk pushes, the
streamed real-time factor (GPU time of all pushes, and the flush, whose own latency is reported too, over the audio's duration at 22050 Hz: below 1 is
faster than real time; 24000 Hz for the U-Net HiFi-GAN and the VQ-VAE, 16000 Hz for the discrete-symbol HiFi-GAN), the libpwgb kernel launches of one steady-state eager push (the few torch copies are not
counted), the stream's state_bytes() and algorithmic latency (delay plus one chunk, in ms at 22050 Hz), and the
whole-utterance forward of the same audio (one call on the B utterances; for MB-MelGAN with the PQMF
synthesis) for comparison.

Every timed stream is checked against ``model.inference`` of each item in the same run:

* pwg, pwg_centred: bit for bit while a push (for pwg_centred also its 16-frame flush push) has at most 65536 samples
  in all (B x chunk x 256), so that its 64 -> 1 output conv takes conv1d_small_cout_kernel as the per-item inference
  does; above that the push's output conv takes conv1d_fewcout_long_kernel, which sums in another order, and the check
  is rel-L2 <= 1e-6;
* hifigan, hifigan_centred (after its delay): the per-item inference's 32 -> 1 output conv has 65536 output samples and takes conv1d_fewcout_long_kernel,
  which sums in another order than the generic kernel every stream conv takes, so the check is rel-L2 <= 1e-6 (bit
  identity holds up to 15 frames, tests/test_gpu_hifigan_stream.py);
* melgan_v1, mb_melgan_v2 and their centred forms: after the delay, the per-item inference's output conv has 67328 output samples and
  takes conv1d_fewcout_long_kernel too, so the check is rel-L2 <= 1e-6 (bit identity holds below 4096 output-conv
  samples, tests/test_gpu_melgan_stream.py);
* uhifigan_opencpop_centred: its inference's 32 -> 1 output conv has 76800 samples and takes conv1d_fewcout_long_kernel,
  so the check is rel-L2 <= 1e-6 (bit identity holds below 4096 samples, tests/test_gpu_uhifigan_lookahead_stream.py);
* vqvae_vctk_lg: against decode(encode(x), l, g) of the batch, whose 32 -> 1 output conv has 16384 samples per item and
  takes conv1d_fewcout_long_kernel, so the check is rel-L2 <= 1e-6 (bit identity holds below 4096 samples,
  tests/test_gpu_vqvae_lookahead_stream.py);
* dsym_vctk_centred: its inference's 32 -> 1 output conv has 81920 samples and takes conv1d_fewcout_long_kernel, so the
  check is rel-L2 <= 1e-6 (bit identity holds below 4096 samples, tests/test_gpu_dsym_lookahead_stream.py);
* dsym_dur_cvss: durations equal ``synthesis``'s exactly, and the audio is within rel-L2 1e-6 of it (its output conv
  takes conv1d_fewcout_long_kernel at this length).

Prints the card name and power limit of the same run, as one JSON document.

    python tools/stream_bench.py [MODEL] [B ...]        # default: every model at B = 1 16"""
import argparse
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
from parallelwavegan_b200.streaming import (CausalHiFiGANStream, CausalMelGANStream, CausalPWGStream,  # noqa: E402
                                            DiscreteSymbolHiFiGANLookaheadStream, HiFiGANLookaheadStream, MelGANLookaheadStream, PWGLookaheadStream, UHiFiGANLookaheadStream, VQVAELookaheadStream)

MELGAN = {
    "melgan_v1": dict(in_channels=80, out_channels=1, kernel_size=7, channels=512, upsample_scales=[8, 8, 2, 2], stacks=3,
                      use_causal_conv=True),
    "mb_melgan_v2": dict(in_channels=80, out_channels=4, kernel_size=7, channels=384, upsample_scales=[8, 4, 2], stacks=4,
                         use_causal_conv=True),
}
MELGAN.update({f"{k}_centred": dict(v, use_causal_conv=False) for k, v in list(MELGAN.items())})
UHIFIGAN_OPENCPOP = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[5, 5, 4, 3],
                         downsample_kernel_sizes=[10, 10, 8, 6], upsample_scales=[3, 4, 5, 5], upsample_kernel_sizes=[6, 8, 10, 10],
                         resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3)
# egs/vctk/vq1/conf/local_conditioned_melgan_vae.v3.yaml generator_params
VQVAE_VCTK_LG = dict(in_channels=1, out_channels=1, num_embeds=512, embed_dim=256, num_local_embeds=2, local_embed_dim=32,
                     num_global_embeds=128, global_embed_dim=128, encoder_type="MelGANDiscriminator", decoder_type="MelGANGenerator",
                     encoder_conf={"out_channels": 256, "downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 1024},
                     decoder_conf={"in_channels": 416, "upsample_scales": [4, 4, 2, 2], "channels": 512, "stacks": 3})
# egs/vctk/hubert_voc1 generator_params (DiscreteSymbolHiFiGANGenerator)
DSYM_VCTK = dict(in_channels=512, out_channels=1, channels=512, num_embs=100, num_spk_embs=128, spk_emb_dim=512, kernel_size=7,
                 upsample_scales=[10, 8, 2, 2], upsample_kernel_sizes=[20, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11],
                 resblock_dilations=[[1, 3, 5]] * 3)
DSYM_DUR_CVSS = dict(in_channels=512, out_channels=1, channels=512, num_embs=500, num_spk_embs=0, kernel_size=7,
                     upsample_scales=[10, 8, 2, 2], upsample_kernel_sizes=[20, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11],
                     resblock_dilations=[[1, 3, 5]] * 3)
MODELS = ("pwg", "pwg_centred", "hifigan", "hifigan_centred", *MELGAN, "uhifigan_opencpop_centred", "vqvae_vctk_lg",
          "dsym_vctk_centred", "dsym_dur_cvss")
FRAMES = 256
CHUNKS = (1, 4, 16, 64)
PASSES = 2
SR = 22050
CHUNKS_OF = {"uhifigan_opencpop_centred": (1, 8), "vqvae_vctk_lg": (1, 4, 16), "dsym_vctk_centred": (1, 4, 16)}
SR_OF = {"uhifigan_opencpop_centred": 24000, "vqvae_vctk_lg": 24000, "dsym_vctk_centred": 16000}


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
    if name == "pwg":
        m, scale = models.ParallelWaveGANGenerator(use_causal_conv=True), 1.0
    elif name == "pwg_centred":
        m, scale = models.ParallelWaveGANGenerator(use_causal_conv=False), 1.0
    elif name == "hifigan":
        m, scale = models.HiFiGANGenerator(use_causal_conv=True), 1.15
    elif name == "hifigan_centred":
        m, scale = models.HiFiGANGenerator(use_causal_conv=False), 1.15
    elif name == "uhifigan_opencpop_centred":
        m, scale = models.UHiFiGANGenerator(**UHIFIGAN_OPENCPOP), 1.15
    elif name == "vqvae_vctk_lg":
        m, scale = models.VQVAE(**VQVAE_VCTK_LG), 1.15
    elif name == "dsym_vctk_centred":
        m, scale = models.DiscreteSymbolHiFiGANGenerator(**DSYM_VCTK), 1.15
    else:
        m, scale = models.MelGANGenerator(**MELGAN[name]), 1.0
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, scale))
    m.remove_weight_norm()
    m = m.eval().to(dev)
    if name in MELGAN and MELGAN[name]["out_channels"] > 1:
        m.pqmf = PQMF(MELGAN[name]["out_channels"]).to(dev)
    return m


class Workload:
    """One model's utterance: its inputs, reference, whole-utterance forward, streams and pushes"""

    def __init__(self, name, m, B, dev):
        self.name, self.m = name, m
        self.melgan = name in MELGAN
        self.flushes = self.melgan or name.endswith("_centred") or name == "vqvae_vctk_lg"
        self.open = 7 if self.melgan and MELGAN[name]["use_causal_conv"] else 0
        self.frames = self.open + FRAMES
        g = torch.Generator().manual_seed(B)
        c = self.c = torch.randn(B, self.frames, 80, generator=g).to(dev)
        cw = c.transpose(1, 2).contiguous()
        self.delay, self.hop, self.sr = 0, 256, SR_OF.get(name, SR)
        if name == "uhifigan_opencpop_centred":
            hop = self.hop = 300
            e = self.e = torch.randn(B, FRAMES * hop, generator=g).to(dev) * 0.3
            self.delay = UHiFiGANLookaheadStream(m, batch=B, use_graphs=False).delay
            self.ref = F.pad(torch.stack([m.inference(excitation=e[b], c=c[b]).t() for b in range(B)]), (self.delay, 0))
            self.whole = lambda: m(cw, None, e.unsqueeze(1))
        elif name == "vqvae_vctk_lg":
            hop = self.hop = 64
            x = self.x = torch.randn(B, 1, FRAMES * hop, generator=g).to(dev) * 0.5
            self.l = torch.randn(B, 2, FRAMES, generator=g).to(dev)
            self.g = torch.arange(B, device=dev) * 7 % 128  # a different target speaker per slot
            self.delay = VQVAELookaheadStream(m, batch=B, use_graphs=False).delay
            self.whole = lambda: m.decode(m.encode(x), self.l, self.g)
            self.ref = F.pad(self.whole(), (self.delay, 0))
        elif name == "dsym_vctk_centred":
            self.hop = 320
            sym = torch.randint(0, DSYM_VCTK["num_embs"], (B, self.frames), generator=g)
            spk = (torch.arange(B) * 7 % DSYM_VCTK["num_spk_embs"])[:, None].expand(B, self.frames)  # a speaker per slot
            c = self.c = torch.stack([sym, spk], -1).to(dev)  # (B, T, 2) units and speaker ids
            cu = c.transpose(1, 2).contiguous()
            self.delay = DiscreteSymbolHiFiGANLookaheadStream(m, batch=B, use_graphs=False).delay
            self.ref = F.pad(torch.stack([m.inference(c[b]).t() for b in range(B)]), (self.delay, 0))
            self.whole = lambda: m(cu)
        elif name in ("pwg", "pwg_centred"):
            hop = self.hop = m.upsample_factor
            z = self.z = torch.randn(B, 1, FRAMES * hop, generator=g).to(dev)
            self.ref = torch.stack([m.inference(c=c[b], x=z[b].t()).t() for b in range(B)])
            if name == "pwg_centred":
                self.delay = PWGLookaheadStream(m, batch=B, use_graphs=False).delay
                self.ref = F.pad(self.ref, (self.delay, 0))
            # the inference input: edge-padded by aux_context_window
            acw = m.aux_context_window
            cw = cw[:, :, torch.arange(-acw, FRAMES + acw, device=dev).clamp(0, FRAMES - 1)].contiguous()
            self.whole = lambda: m(z, cw)
        elif name == "hifigan":
            self.ref = torch.stack([m.inference(c[b]).t() for b in range(B)])
            self.whole = lambda: m(cw)
        elif name == "hifigan_centred":
            self.delay = HiFiGANLookaheadStream(m, batch=B, use_graphs=False).delay
            self.ref = F.pad(torch.stack([m.inference(c[b]).t() for b in range(B)]), (self.delay, 0))
            self.whole = lambda: m(cw)
        else:
            probe = self.stream(B, False)
            assert not self.open or probe.min_first_frames == self.open, probe.min_first_frames
            self.delay = probe.delay
            self.ref = F.pad(torch.stack([m.inference(c[b]).t() for b in range(B)]), (self.delay, 0))
            self.whole = lambda: m.pqmf.synthesis(m(cw)) if m.pqmf is not None else m(cw)
        self.samples = self.ref.shape[-1] - self.delay

    def stream(self, B, graphs):
        cls = {"pwg": CausalPWGStream, "pwg_centred": PWGLookaheadStream, "hifigan": CausalHiFiGANStream,
               "hifigan_centred": HiFiGANLookaheadStream, "uhifigan_opencpop_centred": UHiFiGANLookaheadStream,
               "vqvae_vctk_lg": VQVAELookaheadStream, "dsym_vctk_centred": DiscreteSymbolHiFiGANLookaheadStream}.get(self.name)
        if cls is None:
            cls = CausalMelGANStream if MELGAN[self.name]["use_causal_conv"] else MelGANLookaheadStream
        return cls(self.m, batch=B, use_graphs=graphs)

    def push(self, st, j, n):
        if self.name in ("pwg", "pwg_centred"):
            return st.push(self.c[:, j:j + n], self.z[:, :, j * self.hop:(j + n) * self.hop])
        if self.name == "uhifigan_opencpop_centred":
            return st.push(self.c[:, j:j + n], self.e[:, j * self.hop:(j + n) * self.hop])
        if self.name == "vqvae_vctk_lg":
            return st.push(self.x[..., j * self.hop:(j + n) * self.hop], self.l[..., j:j + n], self.g)
        return st.push(self.c[:, j:j + n])

    def check(self, s, B, n):
        flush_frames = -(-self.delay // self.hop) if self.name == "pwg_centred" else 0
        if self.name in ("pwg", "pwg_centred") and B * max(n, flush_frames) * self.hop <= 65536:
            assert s["bit_identical_to_inference"], (self.name, B, n)
        else:
            assert s["rel_l2_vs_inference"] <= 1e-6, (self.name, B, n, s["rel_l2_vs_inference"])


def bench_model(name, Bs, dev):
    m = build(name, dev)
    res = {}
    for B in Bs:
        w = Workload(name, m, B, dev)
        res.update(frames=w.frames, opening_push_frames=w.open)
        for _ in range(3):
            w.whole()
        row = {"samples_per_item": w.samples, "delay_samples": w.delay,
               "whole_utterance_forward": stats([timed(w.whole)[1] for _ in range(5)])}
        audio_s = w.samples / w.sr
        for graphs in (False, True):
            for n in CHUNKS_OF.get(name, CHUNKS):
                st = w.stream(B, graphs)
                if w.open:  # warm-up: caches, weight packing, graph capture of every length
                    w.push(st, 0, w.open)
                w.push(st, w.open, n)
                capi.reset_launch_count()
                w.push(st, w.open + n, n)
                launches = capi.launch_count()  # a steady-state push (0 with graphs: the replay launches nothing)
                row["state_bytes_per_slot"] = st.state_bytes()
                lat, flushes, total = [], [], 0.0
                for _ in range(PASSES):
                    st.reset()
                    ys = []
                    if w.open:
                        y, t = timed(lambda: w.push(st, 0, w.open))
                        ys.append(y)
                        total += t
                    for j in range(w.open, w.frames, n):
                        y, t = timed(lambda: w.push(st, j, n))
                        lat.append(t)
                        total += t
                        ys.append(y)
                    if w.flushes:
                        y, t = timed(st.flush)
                        flushes.append(t)
                        total += t
                        ys.append(y)
                y = torch.cat(ys, -1)
                s = stats(lat)
                s["rtf"] = total / PASSES / 1e3 / audio_s
                s["algorithmic_latency_ms"] = (w.delay + n * w.hop) / w.sr * 1e3
                if flushes:
                    s["flush_ms"] = sorted(flushes)[len(flushes) // 2]  # every slot at once; the upper median of the passes
                if not graphs:
                    s["libpwgb_launches_per_push"] = launches
                s["bit_identical_to_inference"] = torch.equal(y, w.ref)
                s["rel_l2_vs_inference"] = float((y - w.ref).double().norm() / w.ref.double().norm())
                row[f"{'graph' if graphs else 'eager'}_chunk{n}"] = s
                w.check(s, B, n)
        res[f"B{B}"] = row
    return res


def bench_duration(Bs, dev):
    """dsym_dur_cvss: push latency per push of units, RTF over the audio the pushes and flush produce"""
    from parallelwavegan_b200.streaming import DiscreteSymbolDurationLookaheadStream

    m = models.DiscreteSymbolDurationGenerator(**DSYM_DUR_CVSS)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.15))
    m.remove_weight_norm()
    with torch.no_grad():
        m.duration_predictor.linear.bias.fill_(0.6)
    m = m.eval().to(dev)
    res, S, sr = {}, 128, 16000
    for B in Bs:
        g = torch.Generator().manual_seed(B)
        c = torch.randint(0, DSYM_DUR_CVSS["num_embs"], (B, S), generator=g).to(dev)
        refs = [m.synthesis(c[b:b + 1, None]) for b in range(B)]
        row = {"units_per_item": S}
        for graphs in (False, True):
            for n in (1, 4, 16):
                st = DiscreteSymbolDurationLookaheadStream(m, batch=B, use_graphs=graphs)
                for j in range(0, S, n):  # warm-up pass: caches and every captured length
                    st.push(c[:, j:j + n])
                st.flush()
                lat, total, outs, durs = [], 0.0, [[] for _ in range(B)], [[] for _ in range(B)]
                for j in range(0, S, n):
                    y, t = timed(lambda: st.push(c[:, j:j + n]))
                    lat.append(t)
                    total += t
                    d = st.last_durations
                    for b in range(B):
                        outs[b].append(y[b])
                        durs[b].append(d[b])
                fl, t = timed(st.flush)
                total += t
                d = st.last_durations
                err, same = 0.0, True
                for b in range(B):
                    y = torch.cat(outs[b] + [fl[b]], -1)[:, st.delay:]
                    same &= torch.equal(torch.cat(durs[b] + [d[b]]), refs[b][1][0].cpu())
                    r = refs[b][0][0]
                    err = max(err, float((y - r).double().norm() / r.double().norm()))
                assert same and err <= 1e-6, (B, n, same, err)
                s = stats(lat)
                audio_s = sum(int(r[1].sum()) for r in refs) / B * 320 / sr
                s.update(rtf=total / 1e3 / audio_s, flush_ms=t, durations_equal_synthesis=same, rel_l2_vs_synthesis=err,
                         delay_samples=st.delay, state_bytes_per_slot=st.state_bytes())
                row[f"{'graph' if graphs else 'eager'}_units{n}"] = s
        res[f"B{B}"] = row
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0], formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("model", nargs="?", choices=MODELS, help="the model to stream (default: every one)")
    ap.add_argument("batch", nargs="*", type=int, default=[1, 16], help="batch sizes (default: 1 16)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"card": card(), "sample_rate_for_rtf": SR}
    with torch.no_grad():
        for name in [a.model] if a.model else MODELS:
            out[name] = bench_duration(a.batch, dev) if name == "dsym_dur_cvss" else bench_model(name, a.batch, dev)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
