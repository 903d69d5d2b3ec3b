"""The lifecycle every chunk stream shares, checked once per stream class: batch slots are independent (B = 4 equals four
B = 1 streams), graph replay equals eager runs, a mid-stream reset or a one-slot flush leaves the other slots
bit-identical, more chunk lengths than are cached still match, ``state_bytes`` counts ``_state()``, and the models a
stream cannot take raise ``PwgbError`` naming the stream.  What each stream computes is checked against its oracle and
``inference`` in its own test file."""
import json

import pytest
import torch

from helpers import load_golden
from oracle import synth
from stream_harness import dev, golden_model, synthetic_model  # noqa: F401

pytestmark = pytest.mark.gpu

PWG = dict(in_channels=1, out_channels=1, kernel_size=3, layers=30, stacks=3, residual_channels=64, gate_channels=128,
           skip_channels=64, aux_channels=80, aux_context_window=2, upsample_conditional_features=True,
           upsample_net="ConvInUpsampleNetwork", upsample_params={"upsample_scales": [4, 4, 4, 4]})
DSYM = dict(in_channels=32, out_channels=1, channels=64, num_embs=50, num_spk_embs=4, spk_emb_dim=32, kernel_size=7,
            upsample_scales=[12, 10, 2, 2], upsample_kernel_sizes=[24, 20, 4, 4], resblock_kernel_sizes=[3, 7, 11],
            resblock_dilations=[[1, 3, 5]] * 3)
DUR = dict(in_channels=48, out_channels=1, channels=64, num_embs=30, num_spk_embs=0, duration_chans=64, kernel_size=7,
           upsample_scales=[4, 2], upsample_kernel_sizes=[8, 4], resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])


def _pwg(causal):
    return lambda dev: synthetic_model(dev, "ParallelWaveGANGenerator", dict(PWG, use_causal_conv=causal), 81, 1.0)


def _golden(cls, name):
    return lambda dev: golden_model(dev, cls, name)[2]


def _vqvae(dev):
    from parallelwavegan_b200 import models
    from test_vqvae_cpu import vq_weights

    meta, _ = load_golden("vqvae_yesno")
    m = models.VQVAE(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(vq_weights(meta, fold=False))
    return m.to(dev).eval()


def _duration(dev):
    m = synthetic_model(dev, "DiscreteSymbolDurationGenerator", DUR, 41, 1.15)
    with torch.no_grad():
        m.duration_predictor.linear.bias.fill_(1.2)  # durations of 0 .. 6 frames
    return m


def _mels(st, B, n, seed):
    return (synth.randn((B, n, st.in_channels), seed),)


def _mels_noise(st, B, n, seed):
    return synth.randn((B, n, st.A), seed), synth.randn((B, 1, n * st.hop), seed + 1)


def _mels_excitation(st, B, n, seed):
    return synth.randn((B, n, st.in_channels), seed), synth.randn((B, n * st.hop), seed + 1, 0.3)


def _audio(st, B, n, seed):
    return (synth.randn((B, n * st.hop), seed, 0.3),)


def _units(st, B, n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.stack([torch.randint(0, 50, (B, n), generator=g), torch.randint(0, 4, (B, n), generator=g)], -1),)


def _symbols(st, B, n, seed):
    return (torch.randint(0, DUR["num_embs"], (B, n), generator=torch.Generator().manual_seed(seed)),)


# stream class: (model factory, the inputs of one push of n frames for B slots, whether the stream has a flush)
ROWS = {
    "CausalPWGStream": (_pwg(True), _mels_noise, False),
    "PWGLookaheadStream": (_pwg(False), _mels_noise, True),
    "CausalHiFiGANStream": (_golden("HiFiGANGenerator", "hifigan_causal"), _mels, False),
    "HiFiGANLookaheadStream": (_golden("HiFiGANGenerator", "hifigan_small"), _mels, True),
    "DiscreteSymbolHiFiGANLookaheadStream":
        (lambda dev: synthetic_model(dev, "DiscreteSymbolHiFiGANGenerator", DSYM, 31, 1.15), _units, True),
    "DiscreteSymbolDurationLookaheadStream": (_duration, _symbols, True),
    "CausalMelGANStream": (_golden("MelGANGenerator", "melgan_causal_zero"), _mels, True),
    "MelGANLookaheadStream": (_golden("MelGANGenerator", "melgan_small"), _mels, True),
    "VQVAELookaheadStream": (_vqvae, _audio, True),
    "UHiFiGANLookaheadStream": (_golden("UHiFiGANGenerator", "uhifigan_small"), _mels_excitation, True),
}
SCHEDULE = [1, 4, 2, 5, 3, 6]  # the events below happen before push 3, after 7 frames; 14 frames follow them


@pytest.fixture(scope="module")
def built():
    return {}


def _setup(built, dev, name):
    """the stream class and its model, built once per module"""
    from parallelwavegan_b200 import streaming

    if name not in built:
        built[name] = ROWS[name][0](dev)
    return getattr(streaming, name), built[name]


def _pushes(cls, m, B, schedule, seed):
    """the inputs of every push of ``schedule`` for B slots"""
    st = cls(m, batch=1)
    return [ROWS[cls.__name__][1](st, B, n, seed + 10 * i) for i, n in enumerate(schedule)]


def _signals(st, pushes, flush, event=None):
    """Each slot's concatenated output over ``pushes`` (then a flush of every slot, if the stream has one);
    ``event(st)`` runs before push 3."""
    outs = [[] for _ in range(st.B)]
    for i, args in enumerate(pushes):
        if i == 3 and event is not None:
            event(st)
        y = st.push(*args)
        for b in range(st.B):
            outs[b].append(y[b])
    if flush:
        for b, f in enumerate(st.flush()):
            outs[b].append(f)
    return [torch.cat(o, -1) for o in outs]


def _slot(args, b):
    return tuple(a[b:b + 1] for a in args)


@pytest.mark.parametrize("name", list(ROWS))
def test_slots_graphs_reset_and_flush(dev, built, name):
    """B = 4 equals four B = 1 streams and eager equals graph replay, bit for bit; a mid-stream reset of slot 1 leaves the
    other slots bit-identical; flushing slot 0 mid-stream leaves slot 1's whole output bit-identical"""
    cls, m = _setup(built, dev, name)
    flush = ROWS[name][2]
    pushes = _pushes(cls, m, 4, SCHEDULE, 7)
    y4 = _signals(cls(m, batch=4), pushes, flush)
    for b in range(4):
        y1 = _signals(cls(m, batch=1), [_slot(a, b) for a in pushes], flush)
        assert torch.equal(y1[0], y4[b]), b
    eager = _signals(cls(m, batch=4, use_graphs=False), pushes, flush)
    for b in range(4):
        assert torch.equal(eager[b], y4[b]), b
    reset = _signals(cls(m, batch=4), pushes, flush, lambda st: st.reset(1))
    for b in (0, 2, 3):
        assert torch.equal(reset[b], y4[b]), b
    if flush:
        two = [tuple(a[:2] for a in args) for args in pushes]
        flushed = _signals(cls(m, batch=2), two, flush, lambda st: st.flush(0))
        assert torch.equal(flushed[1], y4[1])


@pytest.mark.parametrize("name", list(ROWS))
def test_more_chunk_lengths_than_cached(dev, built, name):
    """a schedule of MAX_CHUNK_LENGTHS + 2 distinct chunk lengths (cached entries and graphs evicted and rebuilt) equals
    the eager run, bit for bit"""
    cls, m = _setup(built, dev, name)
    sched = list(range(1, cls.MAX_CHUNK_LENGTHS + 3))
    pushes = _pushes(cls, m, 2, sched, 9)
    flush = ROWS[name][2]
    y = _signals(cls(m, batch=2), pushes, flush)
    eager = _signals(cls(m, batch=2, use_graphs=False), pushes, flush)
    for b in range(2):
        assert torch.equal(y[b], eager[b]), b


@pytest.mark.parametrize("name", list(ROWS))
def test_state_bytes(dev, built, name):
    cls, m = _setup(built, dev, name)
    st = cls(m, batch=3)
    assert st.state_bytes() == sum(t[0].numel() * t.element_size() for t in st._state())


@pytest.mark.parametrize("name", list(ROWS))
def test_refusals_name_the_stream(dev, name):
    """a model in train mode, a model on the CPU, batch 0 and a model of another class"""
    from parallelwavegan_b200 import models as M
    from parallelwavegan_b200 import streaming
    from parallelwavegan_b200.capi import PwgbError

    cls = getattr(streaming, name)
    m = ROWS[name][0](dev)
    with pytest.raises(PwgbError, match=name):
        cls(m, batch=0)
    with pytest.raises(PwgbError, match=f"{name}.*train mode"):
        cls(m.train())
    with pytest.raises(PwgbError, match=f"{name}.*CUDA"):
        cls(m.eval().cpu())
    other = M.HiFiGANGenerator(channels=32) if "MelGAN" in name or "VQVAE" in name else M.MelGANGenerator(channels=32, upsample_scales=[4, 4])
    with pytest.raises(PwgbError, match=name):
        cls(other.to(dev).eval())
