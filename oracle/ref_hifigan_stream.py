"""Chunked CPU restatement of streaming a causal HiFi-GAN (TEST INFRASTRUCTURE), on top of the pieces of
``oracle/ref_ops.hifigan_generator``.  It carries the same state as ``parallelwavegan_b200.streaming.CausalHiFiGANStream``,
explicitly and in plain tensors, one history per signal:

* the input conv: its last kernel_size - 1 mel frames (zero for a fresh item, the whole-utterance zero padding);
* each conv-transpose: the last frame of its input; a fresh item replicates its first frame (``ReplicationPad1d``);
* each level input: the largest (k_j - 1) * d_j0 over the blocks whose first dilated conv reads it;
* each later dilated-conv input of a block: (k - 1) * d; each second-conv input: k - 1;
* the output conv: its last kernel_size - 1 input samples.

Every causal conv runs as a valid conv on [the last (k - 1) * d history samples | chunk].  ``whole_utterance`` is the
reference it must equal.  The knobs inject plausible mistakes, so that the tests can show each one is caught:
``dil_short`` (each later dilated-conv history one row short), ``up_zero`` (a fresh item's conv-transpose history zero
instead of replicated) and ``lvl_first_only`` (the shared level history sized for the first block only)."""
import torch
import torch.nn.functional as F

from .ref_ops import hifigan_generator
from .ref_stream import drive, keep


def whole_utterance(w, c, cfg):
    """``HiFiGANGenerator.inference`` for a batch of whole utterances c (B, in_channels, T)."""
    return hifigan_generator(w, c, cfg)


def _causal(x, hist, w, b, d, slope):
    """the causal conv of x given the samples in front of it: the last (k - 1) * d of ``hist`` (zero-extended)"""
    need = (w.shape[-1] - 1) * d
    h = hist[..., max(hist.shape[-1] - need, 0):]
    xp = F.pad(torch.cat([h, x], -1), (need - h.shape[-1], 0))
    return F.conv1d(F.leaky_relu(xp, slope), w, b, dilation=d)


class HiFiGANStreamRef:
    """push(c (B, in_channels, n)) -> (B, out_channels, n * hop), for any n >= 1."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, dil_short=0, up_zero=False, lvl_first_only=False):
        assert cfg.get("use_causal_conv"), cfg
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype = cfg, batch, dtype
        self.dil_short, self.up_zero = dil_short, up_zero
        self.slope = cfg.get("negative_slope", 0.1)
        self.ks, self.dils = list(cfg["resblock_kernel_sizes"]), [list(d) for d in cfg["resblock_dilations"]]
        self.scales = list(cfg["upsample_scales"])
        self.nb = len(self.ks)
        self.extra = cfg.get("use_additional_convs", True)
        K = cfg["kernel_size"]
        ch = [cfg["channels"] // 2 ** i for i in range(len(self.scales) + 1)]
        z = lambda C, H: torch.zeros(batch, C, H, dtype=dtype)  # noqa: E731
        self.cin = z(cfg["in_channels"], K - 1)
        self.up = [z(ch[i], 1) for i in range(len(self.scales))]
        first = [(k - 1) * d[0] for k, d in zip(self.ks, self.dils)]
        self.lvl = [z(ch[i + 1], first[0] if lvl_first_only else max(first)) for i in range(len(self.scales))]
        self.xh = [[[z(ch[i + 1], (k - 1) * d) for d in ds[1:]] for k, ds in zip(self.ks, self.dils)] for i in range(len(self.scales))]
        self.xth = [[[z(ch[i + 1], k - 1) for _ in ds] for k, ds in zip(self.ks, self.dils)] for i in range(len(self.scales))]
        self.out = z(ch[-1], K - 1)
        self.fresh = True

    def push(self, c):
        w, slope = self.w, self.slope
        c = c.to(self.dtype)
        h = _causal(c, self.cin, w["input_conv.conv.weight"], w.get("input_conv.conv.bias"), 1, 1.0)
        self.cin = keep(torch.cat([self.cin, c], -1), self.cin.shape[-1])
        for i, s in enumerate(self.scales):
            hist = h[:, :, :1] if self.fresh and not self.up_zero else self.up[i]
            xp = torch.cat([hist, h], -1)
            self.up[i] = xp[:, :, -1:]
            u = F.conv_transpose1d(F.leaky_relu(xp, slope), w[f"upsamples.{i}.1.deconv.weight"], w.get(f"upsamples.{i}.1.deconv.bias"),
                                   stride=s)[:, :, s:-s]
            cs = 0.0
            for j, (k, ds) in enumerate(zip(self.ks, self.dils)):
                p = f"blocks.{i * self.nb + j}"
                x = u
                for idx, d in enumerate(ds):
                    hx = self.lvl[i] if idx == 0 else self.xh[i][j][idx - 1]
                    if idx > 0:
                        self.xh[i][j][idx - 1] = keep(torch.cat([hx, x], -1), hx.shape[-1], self.dil_short)
                    xt = _causal(x, hx, w[f"{p}.convs1.{idx}.1.conv.weight"], w.get(f"{p}.convs1.{idx}.1.conv.bias"), d, slope)
                    if self.extra:
                        ht = self.xth[i][j][idx]
                        self.xth[i][j][idx] = keep(torch.cat([ht, xt], -1), k - 1)
                        xt = _causal(xt, ht, w[f"{p}.convs2.{idx}.1.conv.weight"], w.get(f"{p}.convs2.{idx}.1.conv.bias"), 1, slope)
                    x = xt + x
                cs = cs + x
            self.lvl[i] = keep(torch.cat([self.lvl[i], u], -1), self.lvl[i].shape[-1])
            h = cs / self.nb
        y = torch.tanh(_causal(h, self.out, w["output_conv.1.conv.weight"], w.get("output_conv.1.conv.bias"), 1, 0.01))
        self.out = keep(torch.cat([self.out, h], -1), self.out.shape[-1])
        self.fresh = False
        return y


def stream(w, c, cfg, schedule, **kw):
    """Run ``HiFiGANStreamRef`` over c (B, in_channels, T) in chunks of ``schedule`` frames (repeated until the utterance is
    used up; the last chunk is cut short) and return the concatenated output."""
    ref = HiFiGANStreamRef(w, cfg, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n]), c.shape[-1], schedule)
