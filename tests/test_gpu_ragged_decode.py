"""Ragged batches on the GPU: the masked ResBlock pairs (pwgb_resblock_pair_ext_forward at 32 / 64 channels,
pwgb_resblock_pair_packed_ext_forward at 128 / 256) against the unmasked pair on each item alone, and
``Decoder(ragged=True)`` against ``model.inference`` of each utterance alone."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from helpers import golden_weights, load_golden, rel_l2
from oracle import synth

pytestmark = pytest.mark.gpu

V1 = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 8, 2, 2],
          upsample_kernel_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


# ------------------------------------------------------------------ the masked pairs

def _pair_alone(ops, x, w1, b1, w2, b2, k, d, out=None, accumulate=False, out_scale=1.0):
    """The unmasked pair on one item: the fused entry, or (t % 4 != 0) the two tensor-core convs it replaces"""
    y = ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=0.1, out=out, accumulate=accumulate,
                          out_scale=out_scale)
    if y is None:
        xt = ops.conv1d(x, w1, b1, dilation=d, padding=(k - 1) // 2 * d, pre_slope=0.1)
        y = ops.conv1d(xt, w2, b2, padding=(k - 1) // 2, pre_slope=0.1, residual=x, out=out, accumulate=accumulate,
                       out_scale=out_scale)
    return y


PAIRS = [(c, k, d) for c in (32, 64, 128, 256) for k in (3, 7, 11) for d in (1, 3, 5)]


@pytest.mark.parametrize("channels,k,d", PAIRS)
def test_masked_pair_matches_each_item_alone(dev, channels, k, d):
    from parallelwavegan_b200 import capi, ops

    T = 512
    lens = [1, 37, 301, T]  # one row, rows not aligned to a tile or to 4, the whole launch
    B = len(lens)
    g = torch.Generator().manual_seed(channels * 100 + k * 10 + d)
    x = torch.randn(B, channels, T, generator=g).to(dev)
    for b, L in enumerate(lens):
        x[b, :, L:] = 0
    w1 = (torch.randn(channels, channels, k, generator=g) * 0.05).to(dev)
    w2 = (torch.randn(channels, channels, k, generator=g) * 0.05).to(dev)
    b1 = (torch.randn(channels, generator=g) * 0.5).to(dev)
    b2 = (torch.randn(channels, generator=g) * 0.5).to(dev)
    d_desc = capi.ResBlockDesc(batch=B, channels=channels, t=T, kernel=k, dilation=d, slope=0.1, out_scale=1.0, accumulate=0)
    L_ = capi.lib()
    if not (L_.pwgb_resblock_pair_supported(C.byref(d_desc)) or L_.pwgb_resblock_pair_packed_supported(C.byref(d_desc))):
        pytest.skip("no fused or packed plan for this pair: the block runs two convs and a mask launch")
    lengths = torch.tensor(lens, dtype=torch.int32, device=dev)
    mask = (torch.zeros_like(lengths), lengths, 1, 0)
    base = torch.randn(B, channels, T, generator=g).to(dev)
    for b, L in enumerate(lens):
        base[b, :, L:] = 0  # accumulate: y is zero on entry outside each signal
    for accumulate, out_scale in ((False, 1.0), (False, 1.0 / 3), (True, 1.0 / 3)):
        out = base.clone() if accumulate else torch.full_like(x, float("nan"))
        y = ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=0.1, out=out, accumulate=accumulate,
                              out_scale=out_scale, mask=mask)
        assert y is out
        for b, L in enumerate(lens):
            xb = x[b : b + 1, :, :L].contiguous()
            ob = base[b : b + 1, :, :L].contiguous() if accumulate else None
            ref = _pair_alone(ops, xb, w1, b1, w2, b2, k, d, out=ob, accumulate=accumulate, out_scale=out_scale)
            assert torch.equal(y[b, :, :L], ref[0]), (b, L, accumulate, out_scale)
            tail = y[b, :, L:]
            assert bool((tail == 0).all()) and not bool(torch.signbit(tail).any()), (b, L, "rows past the end are not +0.0")
    # all-open ends and ext == NULL are the unmasked entry
    ref = ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=0.1)
    open_end = torch.full_like(lengths, 2**31 - 1)
    y = ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=0.1, mask=(torch.zeros_like(lengths), open_end, 1, 0))
    assert torch.equal(y, ref)
    y = torch.empty_like(x)
    pk1, pk2 = ops.packed_weight(w1), ops.packed_weight(w2)
    if L_.pwgb_resblock_pair_supported(C.byref(d_desc)):
        rc = L_.pwgb_resblock_pair_ext_forward(C.byref(d_desc), ops._p(x), ops._p(pk1), ops._p(b1), ops._p(pk2), ops._p(b2), None,
                                               ops._p(y), ops._stream())
    else:
        h = torch.empty_like(x)
        rc = L_.pwgb_resblock_pair_packed_ext_forward(C.byref(d_desc), ops._p(x), ops._p(pk1), ops._p(b1), ops._p(pk2), ops._p(b2),
                                                      None, ops._p(h), ops._p(y), ops._stream())
    capi.check(rc, "resblock pair ext (NULL)")
    assert torch.equal(y, ref)


def test_masked_pair_refuses_a_mask_without_counters(dev):
    from parallelwavegan_b200 import capi, ops

    x = torch.zeros(1, 32, 64, device=dev)
    w = torch.zeros(32, 32, 3, device=dev)
    d = capi.ResBlockDesc(batch=1, channels=32, t=64, kernel=3, dilation=1, slope=0.1, out_scale=1.0, accumulate=0)
    ext = capi.StreamExt(frame=None, end=None, rate=1, lookahead=0, res_hist=None, res_hist_len=0, res_delay=0, edge=0, in_lookahead=0)
    pk = ops.packed_weight(w)
    y = torch.empty_like(x)
    rc = capi.lib().pwgb_resblock_pair_ext_forward(C.byref(d), ops._p(x), ops._p(pk), None, ops._p(pk), None, C.byref(ext), ops._p(y),
                                                   ops._stream())
    assert rc != 0 and "mask" in capi.lib().pwgb_last_error().decode()


# ------------------------------------------------------------------ the decoder

def _v1(dev):
    from parallelwavegan_b200 import models

    m = models.HiFiGANGenerator(**json.loads(json.dumps(V1)))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 7, 1.15))
    m.remove_weight_norm()
    return m.to(dev).eval()


def _golden_model(dev, name):
    from parallelwavegan_b200 import models

    meta, _ = load_golden(name)
    cls = models.DiscreteSymbolHiFiGANGenerator if name.startswith("dsym") else models.HiFiGANGenerator
    m = cls(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    return m.to(dev).eval()


def _out_conv_kernel(cin, K, batch, t):
    """The FFMA kernel of the few-channel output conv at (batch, t) output samples (conv1d_simt.cu's dispatch)"""
    if cin >= 64 and batch * t <= 65536:
        return "small_cout"
    if t >= 4096 and cin * K * 16 <= 40 * 1024:
        return "fewcout_long"
    return "generic"


def _same_out_conv(cin, K, L, batch, t):
    """Whether the output conv computes samples [0, L) of an item in the same order alone (t = L) and in the batch: the
    same FFMA kernel, and for conv1d_fewcout_long_kernel the same interior / edge split of every 1024-sample CTA (an
    interior CTA sums channel-outer, an edge CTA tap-outer).  These are the length-dependent choices on the HiFi-GAN
    path that change a sum order (DESIGN.md §3.14)."""
    k = _out_conv_kernel(cin, K, batch, t)
    if k != _out_conv_kernel(cin, K, 1, L):
        return False
    if k != "fewcout_long":
        return True
    pad = (K - 1) // 2

    def interior(first, n):
        return first - pad >= 0 and first + 1023 + K - 1 - pad < n and first + 1023 < n

    return all(interior(f, L) == interior(f, t) for f in range(0, L, 1024))


def _inputs(m, n, seed, longest):
    """16 utterances: length 1, a repeated length, the longest and random ones"""
    rng = np.random.default_rng(seed)
    lens = [1, longest, 9, 9] + [int(v) for v in rng.integers(2, longest, n - 4)]
    if hasattr(m, "emb"):
        spk = m.num_spk_embs > 0
        utts = []
        for L in lens:
            u = np.stack([rng.integers(0, m.emb.num_embeddings, L), np.full(L, rng.integers(0, max(m.num_spk_embs, 1)))], 1)
            utts.append(u if spk else u[:, :1])
        return utts
    return [rng.standard_normal((L, m.input_conv.in_channels if not m.use_causal_conv else m.input_conv.conv.in_channels))
            .astype(np.float32) for L in lens]


def _alone(m, u, dev):
    with torch.no_grad():
        if hasattr(m, "emb"):
            return m.inference(torch.as_tensor(u, dtype=torch.long, device=dev))
        return m.inference(torch.as_tensor(u, device=dev))


# (model, longest utterance in frames, bucket_frames).  Up to 12 frames padded to a multiple of 4, every output conv
# stays below 4096 samples and takes the generic FFMA kernel alone and in the batch: every waveform must be bit-identical.
# The long sets cross the output conv's length-dependent choices for most items (DESIGN.md §3.14): rel-L2 <= 1e-6 there.
NAMES = ["v1", "hifigan_small", "hifigan_odd", "dsym_vctk", "hifigan_causal"]
CASES = [(n, 12, 4) for n in NAMES] + [("v1", 120, 32), ("hifigan_small", 70, 32), ("hifigan_odd", 70, 32), ("dsym_vctk", 60, 32),
                                      ("hifigan_causal", 70, 32)]


@pytest.mark.parametrize("name,longest,bucket", CASES)
def test_ragged_decoder_equals_inference_alone(dev, name, longest, bucket):
    from parallelwavegan_b200 import decode

    m = _v1(dev) if name == "v1" else _golden_model(dev, name)
    utts = _inputs(m, 16, 5, longest)
    hop = int(np.prod(m.upsample_scales)) if hasattr(m, "upsample_scales") else int(np.prod([u[1].stride[0] for u in m.upsamples]))
    dec = decode.Decoder(m, use_graphs=True, max_batch=16, ragged=True, bucket_frames=bucket)
    got = dec.decode(utts, to_pcm16=False)
    eager = decode.Decoder(m, use_graphs=False, max_batch=16, ragged=True, bucket_frames=bucket).decode(utts, to_pcm16=False)
    pcm = dec.decode(utts, to_pcm16=True)
    Tpad = -(-max(len(u) for u in utts) // bucket) * bucket
    oc = m.output_conv[1]
    oc = getattr(oc, "conv", oc)
    exact, crossed = 0, 0
    for i, u in enumerate(utts):
        ref = _alone(m, u, dev)
        assert got[i].shape == ref.shape, (i, got[i].shape, ref.shape)
        assert torch.equal(got[i], eager[i]), (i, "graph replay differs from eager")
        same = _same_out_conv(oc.in_channels, oc.kernel_size[0], len(u) * hop, len(utts), Tpad * hop)
        qref = decode.pcm16(ref[:, 0].contiguous()).cpu().numpy()
        if same:
            exact += 1
            assert torch.equal(got[i], ref), (name, i, len(u), rel_l2(got[i].cpu(), ref.cpu()))
            assert np.array_equal(pcm[i], qref), (name, i)
        else:
            crossed += 1  # the output conv sums this item's samples in another order alone than in the batch
            assert rel_l2(got[i].cpu(), ref.cpu()) <= 1e-6, (name, i, len(u), rel_l2(got[i].cpu(), ref.cpu()))
            assert np.abs(pcm[i].astype(np.int32) - qref.astype(np.int32)).max() <= 1, (name, i)
    if longest <= 12:
        assert crossed == 0, "a short set must take the same kernels alone and in the batch"
    # rank / world sharding gives the same waveforms
    for r in range(2):
        part = decode.Decoder(m, use_graphs=False, max_batch=16, ragged=True, bucket_frames=bucket, rank=r, world=2).decode(utts, to_pcm16=False)
        assert sorted(part) == list(range(r, len(utts), 2))
        for i, y in part.items():
            ref = _alone(m, utts[i], dev)
            assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6, (name, r, i)


def test_ragged_decoder_small_batches_share_graphs(dev):
    """max_batch 4: four batches of sorted lengths, one graph per (batch, padded length), replayed for another mix"""
    from parallelwavegan_b200 import decode

    m = _golden_model(dev, "hifigan_small")
    utts = _inputs(m, 16, 9, 60)
    dec = decode.Decoder(m, use_graphs=True, max_batch=4, ragged=True, bucket_frames=64)
    a = dec.decode(utts, to_pcm16=False)
    n_graphs = len(dec.runner._graphs)
    utts2 = _inputs(m, 16, 10, 60)
    b = dec.decode(utts2, to_pcm16=False)
    assert len(dec.runner._graphs) <= n_graphs + 4
    for outs, us in ((a, utts), (b, utts2)):
        for i, u in enumerate(us):
            assert rel_l2(outs[i].cpu(), _alone(m, u, dev).cpu()) <= 1e-6, i
