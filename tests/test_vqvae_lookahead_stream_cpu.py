"""Streaming a VQ-VAE's wav2wav conversion without a GPU: the float64 chunked restatement
(oracle/ref_vqvae_lookahead_stream.py) equals [zeros(delay) | decode(encode(x), l, g)] for the stored yesno and vctk
goldens under several push schedules, its delay covers the lookahead float64 autograd measures on the model by less
than one hop, and each plausible mistake it can inject makes it fail."""
import pytest
import torch

from helpers import ORACLE_TOL, load_golden, rel_l2
from oracle import ref_vqvae_lookahead_stream as ref
from test_vqvae_cpu import vq_weights

NAMES = ["vqvae_yesno", "vqvae_vctk_g", "vqvae_vctk_lg"]
SCHEDULES = {"ones": [1], "short": [3], "long": [17], "mixed": [1, 4, 2, 9, 1, 3]}
MISTAKES = ["window_shift", "zero_right_edge", "short_l_delay", "decoder_no_lag", "short_lookahead"]


def _case(name):
    meta, g = load_golden(name)
    w = {k: v.double() for k, v in vq_weights(meta).items()}
    return w, meta["kwargs"], g["x"].double(), g.get("l"), g.get("g"), g


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("sched", list(SCHEDULES))
def test_oracle_matches_goldens(name, sched):
    w, cfg, x, l, gid, g = _case(name)
    l = l.double() if l is not None else None
    y, st = ref.stream(w, x, cfg, SCHEDULES[sched], l=l, g=gid)
    with torch.no_grad():
        whole = ref.whole_utterance(w, x, cfg, l, gid)
    assert st.E == 12 and st.delay == 12 * 64 + st.dec.delay
    assert bool((y[..., :st.delay] == 0).all())
    assert rel_l2(y[..., st.delay:], whole) < 1e-12
    assert rel_l2(y[..., st.delay:].float(), g["decode"]) < ORACLE_TOL


@pytest.mark.parametrize("name", ["vqvae_yesno", "vqvae_vctk_lg"])
def test_delay_against_autograd(name):
    w, cfg, x, l, gid, _ = _case(name)
    st = ref.VQVAELookaheadRef(w, cfg)
    frames = 40
    lw = torch.randn(1, l.shape[1], frames, dtype=torch.float64) if l is not None else None
    measured = ref.measured_lookahead(w, cfg, frames, lw, gid[:1] if gid is not None else None)
    assert measured <= st.delay < measured + st.hop, (measured, st.delay)


@pytest.mark.parametrize("mistake", MISTAKES)
def test_oracle_catches_mistakes(mistake):
    w, cfg, x, l, gid, _ = _case("vqvae_vctk_lg")
    l = l.double()
    with torch.no_grad():
        whole = ref.whole_utterance(w, x, cfg, l, gid)
        z_e = ref.encoder(w, x, cfg)
    worst = 0.0
    for sched in ([3], [1, 4, 2, 9]):
        # the codes absorb small errors of z_e, so the encoder's output is compared too
        y, st = ref.stream(w, x, cfg, sched, l=l, g=gid, **{mistake: True})
        d = st.delay
        worst = max(worst, rel_l2(y[..., d:d + whole.shape[-1]], whole) if y.shape[-1] == d + whole.shape[-1] else 1.0,
                    rel_l2(st.z_e, z_e) if st.z_e.shape == z_e.shape else 1.0)
    assert worst > 1e-6, (mistake, worst)


def test_oracle_encoder_output():
    w, cfg, x, l, gid, _ = _case("vqvae_yesno")
    _, st = ref.stream(w, x, cfg, [1, 4, 2, 9])
    assert rel_l2(st.z_e, ref.encoder(w, x, cfg)) < 1e-12
