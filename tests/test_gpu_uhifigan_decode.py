"""``decode.Decoder`` for the U-Net HiFi-GAN: mels and excitations in batches of equal lengths (``exact=True``) or
zero-padded length buckets (``exact=False``), against ``inference(excitation, c=mel)`` of each utterance, with graph
replay, PCM16 and rank / world sharding."""
import numpy as np
import pytest
import torch

from helpers import rel_l2
from stream_harness import debug_get, golden_model, synthetic_model

pytestmark = pytest.mark.gpu

# egs/opencpop/voc1/conf/uhifigan.v1.yaml generator_params
OPENCPOP = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[5, 5, 4, 3],
                downsample_kernel_sizes=[10, 10, 8, 6], upsample_scales=[3, 4, 5, 5], upsample_kernel_sizes=[6, 8, 10, 10],
                resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], dropout=0.1,
                use_additional_convs=True, bias=True, nonlinear_activation="LeakyReLU",
                nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)
KERNEL_ID = {"generic": 0, "small_cout": 1, "fewcout_long": 2}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _model(dev, name):
    if name == "synthetic_opencpop":
        return synthetic_model(dev, "UHiFiGANGenerator", OPENCPOP, 11, 1.15)
    return golden_model(dev, "UHiFiGANGenerator", name)[2]


def _out_conv_kernel(cin, K, batch, t):
    """The FFMA kernel of the few-channel output conv at (batch, t) output samples (conv1d_simt.cu's dispatch)"""
    if cin >= 64 and batch * t <= 65536:
        return "small_cout"
    if t >= 4096 and cin * K * 16 <= 40 * 1024:
        return "fewcout_long"
    return "generic"


def _same_out_conv(cin, K, L, batch, t):
    """Whether the output conv sums samples [0, L) of an item in the same order alone (t = L) and in a batch padded to
    t: the same FFMA kernel and, for conv1d_fewcout_long_kernel, the same interior / edge split of every 1024-sample CTA
    (the rule of DESIGN.md §3.14)"""
    k = _out_conv_kernel(cin, K, batch, t)
    if k != _out_conv_kernel(cin, K, 1, L):
        return False
    if k != "fewcout_long":
        return True
    pad = (K - 1) // 2

    def interior(first, n):
        return first - pad >= 0 and first + 1023 + K - 1 - pad < n and first + 1023 < n

    return all(interior(f, L) == interior(f, t) for f in range(0, L, 1024))


def _utterances(m, lengths, seed):
    rng = np.random.default_rng(seed)
    hop = int(np.prod(m.upsample_scales))
    mels = [rng.standard_normal((L, m.hidden_conv.in_channels)).astype(np.float32) for L in lengths]
    # (T', hop) and (T' * hop,) layouts both occur
    exc = [(0.3 * rng.standard_normal((L, hop))).astype(np.float32) for L in lengths]
    return mels, [e if i % 2 else e.reshape(-1) for i, e in enumerate(exc)], hop


def _inference(m, mel, exc, dev):
    with torch.no_grad():
        return m.inference(torch.as_tensor(exc, device=dev), c=torch.as_tensor(mel, device=dev))


# (model, lengths in frames): short sets stay below 4096 output samples for the small models; the opencpop sets cross it
SETS = [("uhifigan_small", [1, 12, 9, 9, 5, 12, 7, 9]), ("uhifigan_odd", [2, 9, 9, 4, 13, 9, 6, 1]),
        ("uhifigan_opencpop", [1, 13, 13, 4, 40, 13, 27, 40]), ("synthetic_opencpop", [3, 16, 16, 29, 16, 3, 64, 50])]


@pytest.mark.parametrize("name,lengths", SETS)
def test_exact_decoder_equals_inference(dev, name, lengths):
    from parallelwavegan_b200 import decode

    m = _model(dev, name)
    mels, exc, hop = _utterances(m, lengths, 3)
    dec = decode.Decoder(m, use_graphs=True, max_batch=4, exact=True)
    got = dec.decode(mels, to_pcm16=False, excitations=exc)
    pcm = dec.decode(mels, to_pcm16=True, excitations=exc)
    eager_dec = decode.Decoder(m, use_graphs=False, max_batch=4, exact=True)
    eager = eager_dec.decode(mels, to_pcm16=False, excitations=exc)
    oc = m.output_conv[1]
    cin, K = oc.in_channels, oc.kernel_size[0]
    # the last FFMA launch of the eager decode is the output conv of its last batch: confirm the predicted kernel
    lens = {i: len(x) for i, x in enumerate(mels)}
    Tb, grp = list(eager_dec._groups(lens, list(lens)))[-1]
    assert debug_get(3, 6)[0] == KERNEL_ID[_out_conv_kernel(cin, K, len(grp), Tb * hop)]
    for i, (mel, e) in enumerate(zip(mels, exc)):
        ref = _inference(m, mel, e, dev)
        assert debug_get(3, 6)[0] == KERNEL_ID[_out_conv_kernel(cin, K, 1, len(mel) * hop)]
        assert got[i].shape == ref.shape == (len(mel) * hop, 1), (i, got[i].shape, ref.shape)
        assert torch.equal(got[i], eager[i]), (i, "graph replay differs from eager")
        qref = decode.pcm16(ref[:, 0].contiguous()).cpu().numpy()
        if _same_out_conv(cin, K, len(mel) * hop, lengths.count(len(mel)), len(mel) * hop):
            assert torch.equal(got[i], ref), (name, i, rel_l2(got[i].cpu(), ref.cpu()))
            assert np.array_equal(pcm[i], qref), (name, i)
        else:
            assert rel_l2(got[i].cpu(), ref.cpu()) <= 1e-6, (name, i)
            assert np.abs(pcm[i].astype(np.int32) - qref.astype(np.int32)).max() <= 1, (name, i)
    for r in range(2):
        part = decode.Decoder(m, use_graphs=False, max_batch=4, rank=r, world=2).decode(mels, to_pcm16=False, excitations=exc)
        assert sorted(part) == list(range(r, len(mels), 2))
        for i, y in part.items():
            assert torch.equal(y, eager[i]), (r, i)


@pytest.mark.parametrize("name,lengths", SETS)
def test_bucketed_decoder_equals_padded_inference(dev, name, lengths):
    """exact=False: each utterance at its own length, equal to inference of the utterance zero-padded to its bucket
    (zero frames, zero samples) and cropped"""
    from parallelwavegan_b200 import decode

    m = _model(dev, name)
    mels, exc, hop = _utterances(m, lengths, 4)
    bucket = 8
    dec = decode.Decoder(m, use_graphs=True, max_batch=16, exact=False, bucket_frames=bucket)
    got = dec.decode(mels, to_pcm16=False, excitations=exc)
    pcm = dec.decode(mels, to_pcm16=True, excitations=exc)
    oc = m.output_conv[1]
    cin, K = oc.in_channels, oc.kernel_size[0]
    sizes = {}
    for L in lengths:
        key = -(-L // bucket) * bucket
        sizes[key] = sizes.get(key, 0) + 1
    for i, (mel, e) in enumerate(zip(mels, exc)):
        L = len(mel)
        Tb = -(-L // bucket) * bucket
        assert got[i].shape == (L * hop, 1) and pcm[i].shape == (L * hop,), i
        mel_p = np.concatenate([mel, np.zeros((Tb - L, mel.shape[1]), np.float32)])
        e_p = np.concatenate([e.reshape(-1), np.zeros((Tb - L) * hop, np.float32)])
        ref = _inference(m, mel_p, e_p, dev)[: L * hop]
        if _same_out_conv(cin, K, Tb * hop, sizes[Tb], Tb * hop):
            assert torch.equal(got[i], ref), (name, i, rel_l2(got[i].cpu(), ref.cpu()))
        else:
            assert rel_l2(got[i].cpu(), ref.cpu()) <= 1e-6, (name, i)
        assert np.array_equal(pcm[i], decode.pcm16(got[i][:, 0].contiguous()).cpu().numpy())


def test_decoder_ragged_still_refuses_uhifigan(dev):
    from parallelwavegan_b200 import decode
    from parallelwavegan_b200.capi import PwgbError

    with pytest.raises(PwgbError, match="U-Net"):
        decode.Decoder(_model(dev, "uhifigan_small"), ragged=True)
