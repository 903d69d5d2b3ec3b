"""Ragged VQ-VAE conversion without a GPU: a float64 restatement of the masked batch with each item padded at its own
end (DESIGN.md §3.16) equals the lone ``decode(encode(x))`` of every item, each mistake that the masks and edges guard
against moves some item, and the host logic of ``Decoder.convert``: grouping, per-layer lengths, argument refusals, and
the ``decode`` / ``convert`` kind checks."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden
from oracle import ref_vqvae
from test_vqvae_cpu import vq_weights

NAMES = ["vqvae_yesno", "vqvae_vctk_g", "vqvae_vctk_lg"]
SLOPE = 0.2


def _setup(name):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.VQVAE(**copy.deepcopy(meta["kwargs"]))  # the structure (strides, groups, dilations); weights from w
    w = {k: v.double() for k, v in vq_weights(meta).items()}
    return meta, m, w


# ---------------------------------------------------------------------------------------------------- the restatement
def _edge_rows(x, lens, pad_l, pad_r, edge, batch_end=False):
    """x (B, C, T) -> (B, C, pad_l + T + pad_r): row u of item b reads its own row u inside [0, L_b); outside, the row
    of the reflect edge about L_b (about T with ``batch_end``), or zero"""
    B, Cc, T = x.shape
    out = x.new_zeros(B, Cc, pad_l + T + pad_r)
    u = torch.arange(-pad_l, T + pad_r)
    for b in range(B):
        L = T if batch_end else lens[b]
        v = u.clone()
        if edge == "reflect":
            v = torch.where(u < 0, -u, torch.where(u >= L, 2 * (L - 1) - u, u))
        ok = (v >= 0) & (v < T)
        out[b][:, ok] = x[b][:, v[ok]]
    return out


def _mask(y, lens, on=True):
    if on:
        for b, L in enumerate(lens):
            y[b, :, L:] = 0
    return y


def _conv(x, w, b, lens_in, lens_out, *, pad, edge="zero", stride=1, dilation=1, groups=1, pre=None, post=None, mask=True,
          batch_end=False, residual=None):
    """one ragged conv: the pre-activation, each item padded at its own end, the conv, the post-activation, the mask"""
    if pre is not None:
        x = F.leaky_relu(x, pre)
    y = F.conv1d(_edge_rows(x, lens_in, pad, pad, edge, batch_end), w, b, stride=stride, dilation=dilation, groups=groups)
    if residual is not None:
        y = y + residual
    if post == "lrelu":
        y = F.leaky_relu(y, SLOPE)
    elif post == "tanh":
        y = torch.tanh(y)
    return _mask(y, lens_out, mask)


def ragged_convert(m, w, x, lens, l=None, g=None, mistake=None):
    """the masked, per-item-padded batch in float64: x (B, 1, T) with lens samples per item -> (y, indices)"""
    enc = m.encoder
    n = len(enc.layers)
    edge = "zero" if mistake == "zero_reflect" else "reflect"
    be = mistake == "batch_end"
    L = list(lens)
    h = _conv(x, w["encoder.layers.0.1.weight"], w["encoder.layers.0.1.bias"], L, L, pad=(enc.layers[0][1].kernel_size[0] - 1) // 2,
              edge=edge, post="lrelu", mask=mistake != "drop_enc0", batch_end=be)
    for i in range(1, n - 2):
        c = enc.layers[i][0]
        s = c.stride[0]
        Lo = [v // s if mistake == "floor" else -(-v // s) for v in L]
        h = _conv(h, w[f"encoder.layers.{i}.0.weight"], w[f"encoder.layers.{i}.0.bias"], L, Lo, pad=5 * s, stride=s, groups=c.groups,
                  post="lrelu", mask=mistake != f"drop_strided{i}")
        L = Lo
    c = enc.layers[n - 2][0]
    h = _conv(h, w[f"encoder.layers.{n - 2}.0.weight"], w[f"encoder.layers.{n - 2}.0.bias"], L, L, pad=(c.kernel_size[0] - 1) // 2,
              post="lrelu")
    c = enc.layers[n - 1]
    z = _conv(h, w[f"encoder.layers.{n - 1}.weight"], w[f"encoder.layers.{n - 1}.bias"], L, L, pad=(c.kernel_size[0] - 1) // 2)
    frames = L
    idx = ref_vqvae.quantize(z, w["codebook.embedding.weight"])
    dec = ref_vqvae.assemble(w, ref_vqvae.gather(w["codebook.embedding.weight"], idx), l, g)
    # the decoder: reflect-padded input conv, per level conv-transpose + mask and ResidualStacks, output conv + tanh
    dm = m.decoder
    ks = dm.kernel_size
    L = list(frames)
    h = _conv(dec, w["decoder.melgan.1.weight"], w["decoder.melgan.1.bias"], L, L, pad=(ks - 1) // 2, edge=edge, batch_end=be)
    level = -1
    for j, q in enumerate(dm.melgan):
        p = f"decoder.melgan.{j}"
        if isinstance(q, torch.nn.ConvTranspose1d):
            level += 1
            s = q.stride[0]
            h = F.conv_transpose1d(F.leaky_relu(h, SLOPE), w[p + ".weight"], w[p + ".bias"], stride=s, padding=q.padding[0],
                                   output_padding=q.output_padding[0])
            L = [v * s for v in L]
            h = _mask(h, L, mistake != f"drop_convtr{level}")
        elif type(q).__name__ == "ResidualStack":
            d, k = q.dilation, q.kernel_size
            on = mistake != f"drop_stack{level}"
            t = _conv(h, w[p + ".stack.2.weight"], w[p + ".stack.2.bias"], L, L, pad=(k - 1) // 2 * d, edge=edge, dilation=d, pre=SLOPE,
                      mask=on, batch_end=be)
            sk = _conv(h, w[p + ".skip_layer.weight"], w[p + ".skip_layer.bias"], L, L, pad=0, mask=on)
            h = _conv(t, w[p + ".stack.4.weight"], w[p + ".stack.4.bias"], L, L, pad=0, pre=SLOPE, residual=sk, mask=on)
    j = len(dm.melgan) - 2
    y = _conv(h, w[f"decoder.melgan.{j}.weight"], w[f"decoder.melgan.{j}.bias"], L, L, pad=(ks - 1) // 2, edge=edge, pre=SLOPE,
              post="tanh", batch_end=be)
    return y, idx, frames, z


def _batch(m, w, meta, lens, seed):
    hop = m.hop
    T = max(-(-max(lens) // hop) * hop, hop)
    T = -(-T // (4 * hop)) * 4 * hop
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(len(lens), 1, T, generator=g, dtype=torch.float64) * 0.3
    for b, L in enumerate(lens):
        x[b, 0, L:] = 5.0  # garbage past each end: a mask or an edge that reads it shows
    F_ = T // hop
    l = torch.randn(len(lens), m.local_embed.in_channels, F_, generator=g, dtype=torch.float64) if hasattr(m, "local_embed") else None
    gid = torch.tensor([(7 * b + 3) % m.global_embed.num_embeddings for b in range(len(lens))]) if hasattr(m, "global_embed") else None
    return x, l, gid


def _lengths(m):
    """1 sample over the reflect minimum, lengths that are and are not multiples of the hop, the full padded length"""
    hop, least = m.hop, m.min_ragged_samples()
    return [least, least + 1, 4 * hop, 5 * hop + 17, 8 * hop - 1, 12 * hop]


@pytest.mark.parametrize("name", NAMES)
def test_ragged_restatement_matches_lone(name):
    meta, m, w = _setup(name)
    cfg = meta["kwargs"]
    lens = _lengths(m)
    x, l, gid = _batch(m, w, meta, lens, 1)
    assert x.shape[-1] == lens[-1]  # the longest item fills the padded batch
    with torch.no_grad():
        y, idx, frames, _ = ragged_convert(m, w, x, lens, l, gid)
        for b, L in enumerate(lens):
            xb = x[b : b + 1, :, :L]
            ri = ref_vqvae.vqvae_encode(w, xb, cfg)
            Fb = ri.shape[-1]
            assert Fb == frames[b] == -(-L // m.hop)
            assert torch.equal(idx[b, :Fb], ri[0])
            lb = l[b : b + 1, :, :Fb] if l is not None else None
            gb = gid[b : b + 1] if gid is not None else None
            ry = ref_vqvae.vqvae_decode(w, ri, cfg, lb, gb)
            err = float((y[b, :, : Fb * m.hop] - ry[0]).abs().max())
            assert err < 1e-12, (b, L, err)
            assert bool((y[b, :, Fb * m.hop :] == 0).all())


def _mistakes(m):
    n = len(m.encoder.layers)
    levels = sum(isinstance(q, torch.nn.ConvTranspose1d) for q in m.decoder.melgan)
    return (["drop_enc0", "batch_end", "zero_reflect", "floor"] + [f"drop_strided{i}" for i in range(1, n - 2)]
            + [f"drop_stack{i}" for i in range(levels - 1)])


@pytest.mark.parametrize("name", NAMES)
def test_each_mistake_moves_some_item(name):
    """dropping any one mask (the input conv, a strided conv, a level's stacks that the next conv-transpose reads),
    reflecting at the batch's end, zero-padding the reflect convs, or floor lengths changes some item.  A conv-transpose
    mask alone moves nothing here: its only readers are the level's stacks, whose reflect convs stop at the end and
    whose 1x1 convs are pointwise and masked; it guards a decoder with stacks=0 (test_convtr_mask_without_stacks)."""
    meta, m, w = _setup(name)
    lens = _lengths(m)
    x, l, gid = _batch(m, w, meta, lens, 2)
    with torch.no_grad():
        good, _, frames, z_good = ragged_convert(m, w, x, lens, l, gid)
        for mistake in _mistakes(m):
            y, _, _, z = ragged_convert(m, w, x, lens, l, gid, mistake)
            moved = 0.0
            for b, f in enumerate(frames):  # the encoder output (a code may not flip) and the waveform
                moved = max(moved, float((z[b, :, :f] - z_good[b, :, :f]).abs().max()),
                            float((y[b, :, : f * m.hop] - good[b, :, : f * m.hop]).abs().max()))
            assert moved > 1e-6, mistake


def test_convtr_mask_without_stacks():
    """with stacks=0 a level's conv-transpose output is read by the next conv-transpose, which reads one row past the
    end: dropping its mask moves some item"""
    from parallelwavegan_b200 import models

    meta, _ = load_golden("vqvae_yesno")
    kw = copy.deepcopy(meta["kwargs"])
    kw["decoder_conf"] = dict(kw["decoder_conf"], stacks=0)
    torch.manual_seed(0)
    m = models.VQVAE(**kw)
    m.remove_weight_norm()
    w = {k: v.detach().double() for k, v in m.state_dict().items()}
    lens = _lengths(m)
    x, l, gid = _batch(m, w, meta, lens, 3)
    with torch.no_grad():
        good, _, frames, _ = ragged_convert(m, w, x, lens, l, gid)
        bad, _, _, _ = ragged_convert(m, w, x, lens, l, gid, "drop_convtr0")
    moved = max(float((bad[b, :, : f * m.hop] - good[b, :, : f * m.hop]).abs().max()) for b, f in enumerate(frames))
    assert moved > 1e-6


# ---------------------------------------------------------------------------------------------------- host logic
def test_layer_lengths_are_ceil_per_stride():
    _, m, _ = _setup("vqvae_vctk_lg")
    L = torch.tensor([1, 63, 64, 65, 1000], dtype=torch.int32)
    got = m.encoder.layer_lengths(L)
    assert len(got) == len(m.encoder.layers)
    want, cur = [], [1, 63, 64, 65, 1000]
    for f in m.encoder.layers:
        c = f[0] if isinstance(f, torch.nn.Sequential) and isinstance(f[0], torch.nn.Conv1d) else None
        s = c.stride[0] if c is not None else 1
        cur = [-(-v // s) for v in cur]
        want.append(cur)
    assert [t.tolist() for t in got] == want
    assert got[-1].tolist() == [-(-v // m.hop) for v in [1, 63, 64, 65, 1000]]


def test_min_ragged_lengths():
    _, m, _ = _setup("vqvae_vctk_g")
    # vctk: the decoder's input conv needs 4 frames (pad 3); the 9-dilated stacks at 4x (pad 9) need 3; the output conv 1
    assert m.min_ragged_frames() == 4
    assert m.min_ragged_samples() == 3 * m.hop + 1
    _, y, _ = _setup("vqvae_yesno")
    assert y.min_ragged_frames() == 4 and y.min_ragged_samples() == 3 * y.hop + 1


def _bare(model, **kw):
    from parallelwavegan_b200 import decode

    d = object.__new__(decode.Decoder)
    d.model, d.kind = model, decode.decoder_kind(model)
    d.max_batch, d.exact, d.bucket, d.ragged = kw.get("max_batch", 4), kw.get("exact", True), kw.get("bucket", 4), kw.get("ragged", True)
    d.rank, d.world = kw.get("rank", 0), kw.get("world", 1)
    return d


def test_kind_and_refusals():
    from parallelwavegan_b200 import decode, models
    from parallelwavegan_b200.capi import PwgbError

    meta, m, _ = _setup("vqvae_vctk_lg")
    m.eval()
    assert decode.decoder_kind(m) == "wav2wav"
    assert decode.ragged_refusal(m) is None
    with pytest.raises(PwgbError, match="convert"):
        _bare(m).decode([np.zeros((10, 80), np.float32)])
    with pytest.raises(PwgbError, match="not a VQ-VAE"):
        _bare(models.HiFiGANGenerator(channels=32, upsample_scales=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4])).convert([np.zeros(100)])
    with pytest.raises(PwgbError, match="CUDA"):
        decode.Decoder(m, ragged=True)  # a CPU model: no fallback
    pq = models.VQVAE(**dict(copy.deepcopy(meta["kwargs"]), out_channels=2))
    with pytest.raises(PwgbError, match="out_channels > 1"):
        decode._check_wav2wav(pq)
    hop, least = m.hop, m.min_ragged_samples()
    waves = [np.zeros(least + 5, np.float32), np.zeros(3 * hop + 40, np.float32)]
    frames = [-(-len(x) // hop) for x in waves]
    locs = [np.zeros((f, 2), np.float32) for f in frames]
    d = _bare(m)
    for kw, why in [(dict(locals=None, globals=[0, 1]), "locals=.* required"),
                    (dict(locals=locs, globals=None), "globals=.* required"),
                    (dict(locals=locs[:1], globals=[0, 1]), "1 local tracks for 2"),
                    (dict(locals=[locs[0], np.zeros((frames[1] + 1, 2), np.float32)], globals=[0, 1]), "encoder gives"),
                    (dict(locals=locs, globals=[0, 128]), r"speaker id in \[0, 128\)")]:
        with pytest.raises(PwgbError, match=why):
            d.convert(waves, **kw)
    with pytest.raises(PwgbError, match="fewer than"):
        d.convert([np.zeros(least - 1, np.float32)], [np.zeros((-(-(least - 1) // hop), 2), np.float32)], [0])
    with pytest.raises(PwgbError, match=r"\(T,\) or \(T, 1\)"):
        d.convert([np.zeros((least, 2), np.float32)], [np.zeros((frames[0], 2), np.float32)], [0])
    m.train()
    with pytest.raises(PwgbError, match="train mode"):
        d.convert(waves, locs, [0, 1])
    _, g, _ = _setup("vqvae_vctk_g")
    g.eval()
    with pytest.raises(PwgbError, match="no local conditioning"):
        _bare(g).convert(waves, locs, [0, 1])
    _, y, _ = _setup("vqvae_yesno")
    y.eval()
    with pytest.raises(PwgbError, match="no global embedding"):
        _bare(y).convert(waves, None, [0, 1])


def test_convert_groups():
    """ragged runs sort by frames and pad to bucket multiples; exact groups equal sample counts"""
    _, m, _ = _setup("vqvae_yesno")
    d = _bare(m, max_batch=2, bucket=4)
    frames = {0: 9, 1: 4, 2: 30, 3: 5}
    assert list(d._groups(frames, [0, 1, 2, 3])) == [(8, [1, 3]), (32, [0, 2])]
    d = _bare(m, max_batch=4, ragged=False)
    assert list(d._groups({0: 700, 1: 650, 2: 700}, [0, 1, 2])) == [(650, [1]), (700, [0, 2])]


def test_ragged_entry_refusals():
    """the ragged entries refuse a mask without counters, an edge that is not the conv's pad, and a reflect edge on a
    strided conv or with pad >= t_in, before any launch"""
    import __graft_entry__

    __graft_entry__.build()
    from parallelwavegan_b200 import capi

    L = capi.lib()
    cnt = (C.c_int * 2)(3, 4)
    fake = C.c_void_p(256)  # never dereferenced: every call below fails its argument check

    def desc(pad_mode, stride=1, pad=1, t=8):
        t_out = (t + 2 * pad - 3) // stride + 1
        return capi.Conv1dDesc(batch=2, cin=4, cout=4, t_in=t, t_out=t_out, kernel=3, stride=stride, dilation=1, groups=1,
                               pad_left=pad, pad_mode=pad_mode, period=1, t_valid=t, pre_slope=1.0, pre_gate=0, post_act=0,
                               post_slope=0.0, out_scale=1.0, accumulate=0)

    def ext(frame=True, edge=capi.PAD_REFLECT):
        return capi.StreamExt(frame=C.cast(cnt, C.c_void_p) if frame else None, end=C.cast(cnt, C.c_void_p), rate=1, lookahead=0,
                              res_hist=None, res_hist_len=0, res_delay=0, edge=edge, in_lookahead=0)

    cases = [(desc(capi.PAD_REFLECT), ext(frame=False), "counters"),
             (desc(capi.PAD_REFLECT), ext(edge=capi.PAD_ZERO), "pad_mode"),
             (desc(capi.PAD_REFLECT, stride=2), ext(), "stride 1"),
             (desc(capi.PAD_REFLECT, pad=8), ext(), "pad_left"),
             (desc(capi.PAD_ZERO), ext(), "pad_mode")]
    for d, e, why in cases:
        for fn in (L.pwgb_conv1d_ragged_forward, L.pwgb_conv1d_tc_ragged_forward):
            rc = fn(C.byref(d), fake, fake, None, None, C.byref(e), fake, None)
            assert rc == -1 and why in L.pwgb_last_error().decode(), (why, L.pwgb_last_error())
