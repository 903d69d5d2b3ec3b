"""Ragged VQ-VAE conversion on the GPU: the ragged conv entry points (pwgb_conv1d_ragged_forward,
pwgb_conv1d_tc_ragged_forward) against the unmasked call on each item alone at every conv shape of the three VQ-VAE
fixtures, and ``Decoder(vqvae, ragged=True).convert`` against ``decode(encode(x), l, g)`` of each utterance alone."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import load_golden, rel_l2
from test_vqvae_cpu import vq_weights

pytestmark = pytest.mark.gpu
NAMES = ["vqvae_yesno", "vqvae_vctk_g", "vqvae_vctk_lg"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _model(dev, name, weight_norm=True):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.VQVAE(**copy.deepcopy(meta["kwargs"]))
    m.load_state_dict(vq_weights(meta, fold=False))
    if not weight_norm:
        m.remove_weight_norm()
    return meta, g, m.to(dev).eval()


# ---------------------------------------------------------------------------------------------------- entry points
# (cin, cout, kernel, stride, dilation, groups, pad_mode, post): every conv shape of the three fixtures' encoders and
# decoders (the grouped strided convs run through ops.conv1d, which takes the route ``encode`` takes)
CONVS = (
    [(1, 16, 15, 1, 1, 1, "reflect", "lrelu")]  # the encoder's input conv
    + [(ci, co, 10 * s + 1, s, 1, ci // 4, "zero", "lrelu")
       for ci, co, s in [(16, 64, 4), (64, 256, 4), (256, 512, 2), (512, 1024, 2), (16, 32, 4), (32, 32, 4), (32, 32, 2)]]
    + [(1024, 1024, 5, 1, 1, 1, "zero", "lrelu"), (1024, 256, 3, 1, 1, 1, "zero", None),  # the vctk closing convs
       (32, 32, 5, 1, 1, 1, "zero", "lrelu"), (32, 8, 3, 1, 1, 1, "zero", None)]  # the yesno ones
    + [(ci, co, 7, 1, 1, 1, "reflect", None) for ci, co in [(384, 512, ), (416, 512), (8, 64)]]  # decoder input convs
    + [(c, c, 3, 1, d, 1, "reflect", None) for c in (256, 128, 64, 32, 16, 8, 4) for d in (1, 3, 9)]  # stack convs
    + [(c, c, 1, 1, 1, 1, "zero", None) for c in (256, 128, 64, 32, 16, 8, 4)]  # stack 1x1 / skip convs
    + [(c, 1, 7, 1, 1, 1, "reflect", "tanh") for c in (32, 4)]  # the output convs
    + [(16, 16, 3, 1, 1, 1, "replicate", None)]  # the replicate edge
)


def _ids(c):
    return f"ci{c[0]}-co{c[1]}-k{c[2]}-s{c[3]}-d{c[4]}-g{c[5]}-{c[6]}"


@pytest.mark.parametrize("conv", CONVS, ids=_ids)
def test_ragged_conv_matches_each_item_alone(dev, conv):
    """every row inside an item equals the unmasked conv on that item alone (same kernel: every lone length here is
    below the FFMA few-channel kernels' 4096 rows), rows past its end are +0.0, and ext == NULL is the plain call"""
    from parallelwavegan_b200 import ops

    cin, cout, K, s, d, G, pad_mode, post = conv
    pad = (K - 1) // 2 * d if s == 1 else 5 * s
    T = 640 if s == 1 else 160 * s
    # 1 row over the reflect pad (or 1 output row), lengths aligned to no tile or stride, the full launch
    lens = [pad + 1 if pad_mode != "zero" else 1, 37 * s + 3, T * 3 // 4 - 1, T]
    g = torch.Generator().manual_seed(cin * 7 + cout * 3 + K + s + d)
    w = (torch.randn(cout, cin // G, K, generator=g) / (cin // G * K) ** 0.5).to(dev)
    b = (torch.randn(cout, generator=g) * 0.1).to(dev)
    x = torch.randn(len(lens), cin, T, generator=g).to(dev)
    out_lens = [-(-L // s) for L in lens]
    residual = torch.randn(len(lens), cout, T, generator=g).to(dev) if K == 1 else None
    for bi, L in enumerate(lens):
        x[bi, :, L:] = 0 if pad_mode == "zero" else float("nan")  # a reflect edge never reads past the item's end
    kw = dict(stride=s, dilation=d, groups=G, padding=pad, pad_mode=pad_mode, pre_slope=0.2 if s == 1 else 1.0,
              post_act=post, post_slope=0.2)
    mask = (torch.zeros(len(lens), dtype=torch.int32, device=dev), torch.tensor(out_lens, dtype=torch.int32, device=dev), 1, 0)
    with torch.no_grad():
        y = ops.conv1d(x, w, b, residual=residual, mask=mask, **kw)
        for bi, (L, Lo) in enumerate(zip(lens, out_lens)):
            r = residual[bi : bi + 1, :, :Lo].contiguous() if residual is not None else None
            ref = ops.conv1d(x[bi : bi + 1, :, :L].contiguous(), w, b, residual=r, **kw)
            assert ref.shape[-1] == Lo
            assert torch.equal(y[bi, :, :Lo], ref[0]), (bi, L, float((y[bi, :, :Lo] - ref[0]).abs().max()))
            tail = y[bi, :, Lo:]
            assert bool((tail == 0).all()) and not bool(torch.signbit(tail).any()), (bi, L, "rows past the end are not +0.0")
        if pad_mode == "zero":
            for plain, ragged in _null_ext_pairs(torch.nan_to_num(x), w, b, residual, kw):
                assert torch.equal(plain, ragged)


def _null_ext_pairs(x, w, b, residual, kw):
    """each ragged entry with ext == NULL beside the plain entry it must be: (pwgb_conv1d_forward,
    pwgb_conv1d_ragged_forward), and (pwgb_conv1d_tc_forward, pwgb_conv1d_tc_ragged_forward) where the tensor cores
    take the descriptor"""
    from parallelwavegan_b200 import capi, ops

    B, cin, T = x.shape
    cout, _, K = w.shape
    s, d, G, pad = kw["stride"], kw["dilation"], kw["groups"], kw["padding"]
    t_out = (T + 2 * pad - d * (K - 1) - 1) // s + 1
    desc = capi.Conv1dDesc(batch=B, cin=cin, cout=cout, t_in=T, t_out=t_out, kernel=K, stride=s, dilation=d, groups=G,
                           pad_left=pad, pad_mode=capi.PAD_ZERO, period=1, t_valid=T, pre_slope=kw["pre_slope"], pre_gate=0,
                           post_act=ops._ACT[kw["post_act"]], post_slope=kw["post_slope"], out_scale=1.0, accumulate=0)
    lib, a = capi.lib(), (C.byref(desc), ops._p(x))
    tail = (ops._p(b), ops._p(residual))
    outs = [torch.full((B, cout, t_out), float("nan"), device=x.device) for _ in range(4)]
    capi.check(lib.pwgb_conv1d_forward(*a, ops._p(w), *tail, ops._p(outs[0]), ops._stream()), "pwgb_conv1d_forward")
    capi.check(lib.pwgb_conv1d_ragged_forward(*a, ops._p(w), *tail, None, ops._p(outs[1]), ops._stream()), "pwgb_conv1d_ragged_forward")
    pairs = [(outs[0], outs[1])]
    if lib.pwgb_conv1d_tc_supported(C.byref(desc)):
        pk = ops._p(ops.packed_weight(w, G))
        capi.check(lib.pwgb_conv1d_tc_forward(*a, pk, *tail, ops._p(outs[2]), ops._stream()), "pwgb_conv1d_tc_forward")
        capi.check(lib.pwgb_conv1d_tc_ragged_forward(*a, pk, *tail, None, ops._p(outs[3]), ops._stream()), "pwgb_conv1d_tc_ragged_forward")
        pairs.append((outs[2], outs[3]))
    return pairs


# ---------------------------------------------------------------------------------------------------- end to end
def _lone(m, x, l, g):
    with torch.no_grad():
        idx = m.encode(x)
        return idx, m.decode(idx, l, g)


def _corpus(m, meta, n_extra=0, seed=3):
    """waveforms of lengths that are and are not multiples of the hop: 1 sample over the reflect minimum, unaligned,
    aligned, the longest of the run (the batch's full padded length), and one past the FFMA few-channel threshold"""
    hop, least = m.hop, m.min_ragged_samples()
    lens = [least, least + 1, 5 * hop, 7 * hop + 13, 11 * hop - 1, 16 * hop, 4096 + 3 * hop + 5][: 7 + n_extra]
    rng = np.random.default_rng(seed)
    waves = [(0.3 * rng.standard_normal(L)).astype(np.float32) for L in lens]
    locs = None
    if hasattr(m, "local_embed"):
        C_in = m.local_embed.in_channels
        locs = [rng.standard_normal((-(-L // hop), C_in)).astype(np.float32) for L in lens]
    spk = [int(v) for v in rng.integers(0, m.global_embed.num_embeddings, len(lens))] if hasattr(m, "global_embed") else None
    return waves, locs, spk


def _check_against_lone(m, dev, out, waves, locs, spk, items=None):
    hop = m.hop
    for i in (items if items is not None else range(len(waves))):
        y, idx = out[i]
        x = torch.from_numpy(waves[i]).to(dev).reshape(1, 1, -1)
        l = torch.from_numpy(locs[i].T.copy()).to(dev)[None] if locs is not None else None
        g = torch.tensor([spk[i]], device=dev) if spk is not None else None
        ref_idx, ref = _lone(m, x, l, g)
        F = ref_idx.shape[-1]
        assert idx.dtype == np.int64 and idx.shape == (F,) and np.array_equal(idx, ref_idx[0].cpu().numpy()), i
        yy = y[:, 0]
        assert yy.shape[0] == F * hop
        if F * hop < 4096:  # the lone output conv takes the generic FFMA kernel, as the ragged one always does
            assert torch.equal(yy, ref[0, 0]), (i, float((yy - ref[0, 0]).abs().max()))
        else:  # the lone call takes conv1d_fewcout_long_kernel: another sum order
            assert rel_l2(yy, ref[0, 0]) < 1e-6, i


@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_ragged_convert_matches_lone(dev, name, weight_norm):
    from parallelwavegan_b200 import decode

    meta, _, m = _model(dev, name, weight_norm)
    waves, locs, spk = _corpus(m, meta)
    dec = decode.Decoder(m, ragged=True, max_batch=4, bucket_frames=4)
    out = dec.convert(waves, locs, spk, to_pcm16=False)
    assert sorted(out) == list(range(len(waves)))
    _check_against_lone(m, dev, out, waves, locs, spk)
    pcm = dec.convert(waves, locs, spk)
    for i in out:
        ref = decode.pcm16(out[i][0][:, 0].contiguous()).cpu().numpy()
        assert pcm[i][0].dtype == np.int16 and np.array_equal(pcm[i][0], ref) and np.array_equal(pcm[i][1], out[i][1])


def test_ragged_four_speakers_graphs_and_sharding(dev):
    """four target speakers in one batch, graph replay against eager, and rank / world sharding"""
    from parallelwavegan_b200 import decode

    meta, _, m = _model(dev, "vqvae_vctk_g")
    waves, _, _ = _corpus(m, meta)
    waves = waves[:4]
    spk = [0, 5, 17, 99]
    eager = decode.Decoder(m, ragged=True, max_batch=4, bucket_frames=4, use_graphs=False).convert(waves, None, spk, to_pcm16=False)
    _check_against_lone(m, dev, eager, waves, None, spk)
    graphed = decode.Decoder(m, ragged=True, max_batch=4, bucket_frames=4)
    for _ in range(2):  # capture, then replay
        out = graphed.convert(waves, None, spk, to_pcm16=False)
        for i in eager:
            assert torch.equal(out[i][0], eager[i][0]) and np.array_equal(out[i][1], eager[i][1])
    shards = {}
    for rank in range(2):
        part = decode.Decoder(m, ragged=True, max_batch=4, bucket_frames=4, rank=rank, world=2).convert(waves, None, spk, to_pcm16=False)
        assert sorted(part) == [i for i in range(4) if i % 2 == rank]
        shards.update(part)
    for i in eager:
        assert torch.equal(shards[i][0], eager[i][0]) and np.array_equal(shards[i][1], eager[i][1])


@pytest.mark.parametrize("exact", [True, False])
def test_exact_and_padded_convert(dev, exact):
    """exact=True batches equal lengths (each equal to its lone conversion); exact=False pads buckets and crops"""
    from parallelwavegan_b200 import decode

    meta, _, m = _model(dev, "vqvae_vctk_lg")
    waves, locs, spk = _corpus(m, meta)
    waves, locs, spk = waves[:4] + waves[:2], locs[:4] + locs[:2], spk[:4] + spk[:2]
    out = decode.Decoder(m, exact=exact, max_batch=4, bucket_frames=4).convert(waves, locs, spk, to_pcm16=False)
    hop = m.hop
    for i, w in enumerate(waves):
        assert out[i][0].shape == (-(-len(w) // hop) * hop, 1) and out[i][1].shape == (-(-len(w) // hop),)
    if exact:
        _check_against_lone(m, dev, out, waves, locs, spk)


def test_model_ragged_encode_decode(dev):
    """VQVAE.encode / decode with lengths directly: the rows inside each item equal the lone calls, later ones +0.0"""
    meta, _, m = _model(dev, "vqvae_yesno")
    hop = m.hop
    lens = [m.min_ragged_samples(), 9 * hop + 7, 24 * hop]
    T = 24 * hop
    x = torch.zeros(len(lens), 1, T, device=dev)
    g = torch.Generator().manual_seed(5)
    for b, L in enumerate(lens):
        x[b, 0, :L] = (torch.randn(L, generator=g) * 0.3).to(dev)
    with torch.no_grad():
        idx = m.encode(x, torch.tensor(lens, dtype=torch.int32, device=dev))
        frames = [-(-L // hop) for L in lens]
        idx_in = idx.clone()
        for b, F in enumerate(frames):
            idx_in[b, F:] = 0
        y = m.decode(idx_in, lengths=torch.tensor(frames, dtype=torch.int32, device=dev))
        for b, (L, F) in enumerate(zip(lens, frames)):
            ri, ry = _lone(m, x[b : b + 1, :, :L].contiguous(), None, None)
            assert torch.equal(idx[b, :F], ri[0])
            assert torch.equal(y[b, 0, : F * hop], ry[0, 0])
            assert bool((y[b, 0, F * hop :] == 0).all())
