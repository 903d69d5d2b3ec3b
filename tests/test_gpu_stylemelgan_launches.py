"""StyleMelGANGenerator's libpwgb launches per forward and per inference at its golden shapes.  The discrete-symbol
StyleMelGAN shares its noise path and body, so these counts pin that sharing to the launches StyleMelGANGenerator has
always issued: any added, dropped or split launch in the shared code changes them."""
import json

import pytest
import torch

from helpers import golden_weights, load_golden
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


@pytest.mark.parametrize("name,forward_launches,inference_launches", [("style_melgan_small", 62, 62), ("style_melgan_v1", 194, 194)])
def test_launch_counts(dev, name, forward_launches, inference_launches):
    from parallelwavegan_b200 import capi, models

    meta, _ = load_golden(name)
    m = models.StyleMelGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    m = m.to(dev).eval()
    c = synth.randn(meta["c_shape"], meta["c_seed"]).to(dev)
    z = synth.randn(meta["z_shape"], meta["z_seed"]).to(dev)
    ci = synth.randn((100, meta["kwargs"]["aux_channels"]), 5).to(dev)  # T = 100: the conditioning is padded, the output cropped
    noise = synth.randn((1, meta["kwargs"]["in_channels"], -(-100 // m.noise_upsample_factor)), 6).to(dev)
    counts = []
    with torch.no_grad():
        for call in (lambda: m(c, z), lambda: m.inference(ci, noise=noise)):
            call()  # warm-up: weight packing caches
            torch.cuda.synchronize()
            capi.reset_launch_count()
            call()
            torch.cuda.synchronize()
            counts.append(capi.launch_count())
    assert counts == [forward_launches, inference_launches]
