"""Ragged batches without a GPU: a float64 restatement of the length-masked batched HiFi-GAN forward, which masks
exactly where the CUDA path does (the input conv output, each level's conv-transpose output, the ResBlock pair
intermediate and output, each single conv), checked against the forward of each item alone; mutations that drop one
mask each break it, so every mask is needed.  Plus the codegen of the masked pair kernels and the decoder's host
logic (grouping, padding, refusals, argument checks)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from oracle import ref_discrete, ref_ops, synth
from oracle.ref_ops import fold_weight_norm


def _lrelu(x, s):
    return F.leaky_relu(x, s)


def _masked_forward(w, c, lengths, cfg, dsym=False, skip=()):
    """float64 batched forward of a HiFi-GAN body with per-item lengths (frames); ``skip``: masks left out.  c is the
    (B, C, T) input (the embedding for a discrete-symbol model), garbage past each item's end."""
    B, _, T = c.shape

    def mask(x, rate, name):
        if name in skip:
            return x
        x = x.clone()
        for b, L in enumerate(lengths):
            x[b, :, L * rate :] = 0
        return x

    ks, slope = cfg["kernel_size"], 0.1
    nb = len(cfg["resblock_kernel_sizes"])
    if dsym:
        c = mask(c, 1, "embed")
    c = mask(F.conv1d(c, w["input_conv.weight"], w["input_conv.bias"], padding=(ks - 1) // 2), 1, "input")
    rate = 1
    for i, (s, k) in enumerate(zip(cfg["upsample_scales"], cfg["upsample_kernel_sizes"])):
        pad, op = ((k - s) // 2, 0) if dsym else (s // 2 + s % 2, s % 2)
        c = F.conv_transpose1d(_lrelu(c, slope), w[f"upsamples.{i}.1.weight"], w[f"upsamples.{i}.1.bias"], stride=s, padding=pad,
                               output_padding=op)
        rate *= s
        assert c.shape[-1] == T * rate
        c = mask(c, rate, "level")
        cs = 0.0
        for j in range(nb):
            p = f"blocks.{i * nb + j}"
            kk = cfg["resblock_kernel_sizes"][j]
            x = c
            for idx, d in enumerate(cfg["resblock_dilations"][j]):
                xt = F.conv1d(_lrelu(x, slope), w[f"{p}.convs1.{idx}.1.weight"], w.get(f"{p}.convs1.{idx}.1.bias"), dilation=d,
                              padding=(kk - 1) // 2 * d)
                if cfg.get("use_additional_convs", True):
                    xt = mask(xt, rate, "pair_h")
                    xt = F.conv1d(_lrelu(xt, slope), w[f"{p}.convs2.{idx}.1.weight"], w.get(f"{p}.convs2.{idx}.1.bias"),
                                  padding=(kk - 1) // 2)
                    x = mask(xt + x, rate, "pair_out")
                else:
                    x = mask(xt + x, rate, "single")
            cs = cs + x
        c = cs / nb
    c = F.conv1d(_lrelu(c, 0.01), w["output_conv.1.weight"], w["output_conv.1.bias"], padding=(ks - 1) // 2)
    return torch.tanh(c)


SMALL = dict(in_channels=8, out_channels=1, channels=32, kernel_size=7, upsample_scales=[4, 2], upsample_kernel_sizes=[8, 4],
             resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 5]], use_additional_convs=True)
CASES = {
    "v1_small": dict(SMALL),
    "odd_scales": dict(SMALL, upsample_scales=[3, 2], upsample_kernel_sizes=[6, 4]),
    "single_convs": dict(SMALL, use_additional_convs=False),
}
DSYM = dict(in_channels=16, out_channels=1, channels=32, num_embs=20, num_spk_embs=5, spk_emb_dim=16, kernel_size=7,
            upsample_scales=[4, 2], upsample_kernel_sizes=[8, 4], resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 5]])
LENGTHS = [1, 5, 17, 17, 24]  # one frame, a repeated length, the full padded length


def _weights(cls, kw, seed):
    m = cls(**kw)
    return fold_weight_norm(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, 1.15))


def _hifigan_case(name):
    from parallelwavegan_b200 import models

    cfg = CASES[name]
    w = {k: v.double() for k, v in _weights(models.HiFiGANGenerator, cfg, 3).items()}
    g = torch.Generator().manual_seed(4)
    T = max(LENGTHS)
    c = torch.randn(len(LENGTHS), cfg["in_channels"], T, generator=g, dtype=torch.float64)
    for b, L in enumerate(LENGTHS):
        c[b, :, L:] = 0  # zero frames past the end
    return w, c, cfg


def _dsym_case():
    from parallelwavegan_b200 import models

    w = {k: v.double() for k, v in _weights(models.DiscreteSymbolHiFiGANGenerator, DSYM, 5).items()}
    g = torch.Generator().manual_seed(6)
    T = max(LENGTHS)
    sym = torch.randint(0, DSYM["num_embs"], (len(LENGTHS), T), generator=g)
    spk = torch.randint(0, DSYM["num_spk_embs"], (len(LENGTHS),), generator=g)
    for b, L in enumerate(LENGTHS):
        sym[b, L:] = 0  # the decoder pads with symbol 0
    idx = torch.stack([sym, spk[:, None].expand(-1, T)], 1)
    return w, idx, DSYM


def _alone(w, c, cfg, b, L, hifigan=True):
    if hifigan:
        return ref_ops.hifigan_generator(w, c[b : b + 1, :, :L], dict(cfg, negative_slope=0.1))
    return ref_discrete.dsym_generator(w, c[b : b + 1, :, :L], cfg)


def _max_err(y, w, c, cfg, hifigan=True):
    hop = 1
    for s in cfg["upsample_scales"]:
        hop *= s
    err = 0.0
    for b, L in enumerate(LENGTHS):
        ref = _alone(w, c, cfg, b, L, hifigan)
        assert ref.shape[-1] == L * hop
        err = max(err, float((y[b, :, : L * hop] - ref[0]).abs().max() / ref.abs().max()))
    return err


@pytest.mark.parametrize("name", sorted(CASES))
def test_masked_batch_equals_each_item_alone(name):
    w, c, cfg = _hifigan_case(name)
    y = _masked_forward(w, c, LENGTHS, cfg)
    assert _max_err(y, w, c, cfg) < 1e-12


def test_masked_batch_equals_each_item_alone_discrete_symbols():
    w, idx, cfg = _dsym_case()
    y = _masked_forward(w, ref_discrete.embed(w, idx, cfg), LENGTHS, cfg, dsym=True)
    assert _max_err(y, w, idx, cfg, hifigan=False) < 1e-12


@pytest.mark.parametrize("name,drop", [("v1_small", "input"), ("v1_small", "level"), ("v1_small", "pair_h"),
                                       ("v1_small", "pair_out"), ("odd_scales", "level"), ("odd_scales", "pair_h"),
                                       ("single_convs", "single")])
def test_each_mask_is_needed(name, drop):
    w, c, cfg = _hifigan_case(name)
    y = _masked_forward(w, c, LENGTHS, cfg, skip=(drop,))
    assert _max_err(y, w, c, cfg) > 1e-6, f"leaving out the {drop} mask went unnoticed"


def test_discrete_symbol_embed_mask_is_needed():
    w, idx, cfg = _dsym_case()
    y = _masked_forward(w, ref_discrete.embed(w, idx, cfg), LENGTHS, cfg, dsym=True, skip=("embed",))
    assert _max_err(y, w, idx, cfg, hifigan=False) > 1e-6


# ------------------------------------------------------------------ codegen of the masked kernels

def _nvcc():
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.isfile(cand) and os.access(cand, os.X_OK) else None


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parallelwavegan_b200", "csrc")


@pytest.mark.parametrize("src,pattern,count", [("resblock_tc.cu", r"rb_pair_split_ext_kernel", 2),
                                               ("conv1d_tc.cu", r"conv1d_tc_mask_kernel", 1)])
def test_masked_pair_kernels_no_spills_no_serialized_wgmma(tmp_path, src, pattern, count):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path / (src + ".o"))
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
           "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    props = {}
    for m in re.finditer(r"Function properties for (\S*" + pattern + r"\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", r.stdout):
        props[m.group(1)] = tuple(int(g) for g in m.group(2, 3, 4))
    assert len(props) == count, sorted(props)
    assert not {k: v for k, v in props.items() if any(v)}, props
    bad = [line for line in r.stdout.splitlines() if re.search(r"\(C75\d\d\)|serialized", line) and re.search(pattern, line)]
    assert not bad, "\n".join(bad[:10])


# ------------------------------------------------------------------ decoder host logic

def _bare_decoder(**kw):
    from parallelwavegan_b200 import decode

    d = object.__new__(decode.Decoder)
    d.max_batch, d.exact, d.bucket, d.ragged = kw.get("max_batch", 4), kw.get("exact", True), kw.get("bucket", 32), kw.get("ragged", True)
    return d


def test_ragged_groups_sort_by_length_and_pad_to_buckets():
    d = _bare_decoder(max_batch=3, bucket=32)
    lengths = {0: 100, 1: 5, 2: 64, 3: 33, 4: 5, 5: 800, 6: 1}
    groups = list(d._groups(lengths, list(lengths)))
    assert [g for _, g in groups] == [[6, 1, 4], [3, 2, 0], [5]]
    assert [t for t, _ in groups] == [32, 128, 800]
    for t, g in groups:
        assert t % 32 == 0 and t >= max(lengths[i] for i in g)


def test_exact_and_bucketed_groups_unchanged():
    d = _bare_decoder(max_batch=2, ragged=False)
    lengths = {0: 10, 1: 10, 2: 10, 3: 7}
    assert list(d._groups(lengths, [0, 1, 2, 3])) == [(7, [3]), (10, [0, 1]), (10, [2])]
    d = _bare_decoder(max_batch=8, ragged=False, exact=False, bucket=16)
    assert list(d._groups(lengths, [0, 1, 2, 3])) == [(16, [0, 1, 2, 3])]


def test_ragged_refuses_other_generators():
    from parallelwavegan_b200 import decode, models
    from parallelwavegan_b200.capi import PwgbError

    refused = [(models.MelGANGenerator(), "reflection"), (models.ParallelWaveGANGenerator(layers=3, stacks=1), "WaveNet"),
               (models.StyleMelGANGenerator(), "InstanceNorm"), (models.UHiFiGANGenerator(), "U-Net"),
               (models.DiscreteSymbolDurationGenerator(**DSYM), "duration")]
    for m, why in refused:
        with pytest.raises(PwgbError, match=why):
            decode.Decoder(m, ragged=True)
    assert decode.ragged_refusal(models.HiFiGANGenerator(**SMALL)) is None
    assert decode.ragged_refusal(models.HiFiGANGenerator(**dict(SMALL, use_causal_conv=True))) is None
    assert decode.ragged_refusal(models.DiscreteSymbolHiFiGANGenerator(**DSYM)) is None


def test_ragged_argument_checks():
    from parallelwavegan_b200 import decode, models
    from parallelwavegan_b200.capi import PwgbError

    m = models.HiFiGANGenerator(**SMALL)
    with pytest.raises(PwgbError, match="multiple of 4"):
        decode.Decoder(m, ragged=True, bucket_frames=30)
    with pytest.raises(PwgbError, match="positive"):
        decode.Decoder(m, ragged=True, max_batch=0)
    with pytest.raises(PwgbError, match="CUDA"):
        decode.Decoder(m, ragged=True)  # a CPU model: no fallback
    with pytest.raises(PwgbError, match="on the device"):
        models._length_mask(torch.tensor([3, 4], dtype=torch.int32), 2, 1)  # lengths on the host
    with pytest.raises(PwgbError, match=r"\(T, 2\)"):
        decode._unit_rows(torch.zeros(5, 1, dtype=torch.long), speakers=True)
    u = decode._unit_rows([[3, 1], [4, 1]], speakers=False)
    assert u.dtype == torch.int64 and tuple(u.shape) == (2, 1)
