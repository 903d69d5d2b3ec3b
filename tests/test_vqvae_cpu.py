"""VQ-VAE without a GPU: the CPU oracle against the reference's golden outputs and collater batches, and the mirror's
module structure (state-dict names and shapes with and without weight norm, reference-layout loading, the rejected
configurations, loading by config name) against the reference's."""
import numpy as np
import pytest
import torch

from helpers import GOLD, ORACLE_TOL, golden_weights, load_golden, rel_l2
from oracle import ref_vqvae
from oracle.ref_ops import fold_weight_norm

NAMES = ["vqvae_yesno", "vqvae_vctk_g", "vqvae_vctk_lg"]


def vq_weights(meta, fold=True):
    """The fixture's synthetic checkpoint with its codebook scaled as recorded."""
    w = golden_weights(meta)
    w["codebook.embedding.weight"] = w["codebook.embedding.weight"] * meta["codebook_scale"]
    return fold_weight_norm(w) if fold else w


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    meta, g = load_golden(name)
    w, cfg = vq_weights(meta), meta["kwargs"]
    l, gid = g.get("l"), g.get("g")
    with torch.no_grad():
        x_bar, z_e, z_q, idx = ref_vqvae.vqvae_forward(w, g["x"], cfg, l, gid)
        assert torch.equal(idx, g["indices"])
        assert torch.equal(ref_vqvae.vqvae_encode(w, g["x"], cfg), g["indices"])
        for a, b in ((x_bar, g["x_bar"]), (z_e, g["z_e"]), (z_q, g["z_q"])):
            assert rel_l2(a, b) < ORACLE_TOL
        assert rel_l2(ref_vqvae.vqvae_decode(w, g["indices"], cfg, l, gid), g["decode"]) < ORACLE_TOL
    assert meta["min_gap"] >= meta["margin"] >= 1e-3


def test_oracle_collater_matches_reference():
    from oracle.make_golden_vqvae import collate_items

    ref = np.load(f"{GOLD}/vqvae_collate.npz")
    items = collate_items()
    np.random.seed(21)
    (l, g), y = ref_vqvae.collate_vq(items, 1280, 64, 0, use_local_condition=True, use_global_condition=True)
    assert np.array_equal(l, ref["lg_l"]) and np.array_equal(g, ref["lg_g"]) and np.array_equal(y, ref["lg_y"])
    np.random.seed(22)
    (l, g), y = ref_vqvae.collate_vq([(x, gid) for x, _, gid in items], 1280, 64, 0, use_global_condition=True)
    assert l is None and np.array_equal(g, ref["g_g"]) and np.array_equal(y, ref["g_y"])


def _mirror(kwargs, **kw):
    import copy

    from parallelwavegan_b200 import models

    return models.VQVAE(**dict(copy.deepcopy(kwargs), **kw))


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_matches_reference(name):
    meta, _ = load_golden(name)
    m = _mirror(meta["kwargs"])
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, list(s)) for k, s in meta["spec"]]
    m.load_state_dict(vq_weights(meta, fold=False), strict=True)
    if "num_local_embeds" in meta["kwargs"]:
        assert "local_embed.weight_g" in m.state_dict()  # weight-normed like every Conv1d
    if "num_global_embeds" in meta["kwargs"]:
        assert "global_embed.weight" in m.state_dict()  # an Embedding: no weight norm
    m.remove_weight_norm()
    assert not any(k.endswith("weight_g") for k in m.state_dict())
    m.apply_weight_norm()
    assert sorted(m.state_dict()) == sorted(k for k, _ in meta["spec"])


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_without_weight_norm_keeps_the_decoders(name):
    """use_weight_norm=False: the encoder and local_embed are plain, the decoder keeps MelGANGenerator's own weight norm."""
    meta, _ = load_golden(name)
    m = _mirror(meta["kwargs"], use_weight_norm=False)
    keys = list(m.state_dict())
    expect = []
    for k, _ in meta["spec"]:
        if k.startswith("decoder."):
            expect.append(k)
        elif k.endswith(".weight_g"):
            continue
        elif k.endswith(".weight_v"):
            expect.append(k[: -len("_v")])
        else:
            expect.append(k)
    assert sorted(keys) == sorted(expect)
    assert any(k.startswith("decoder.") and k.endswith("weight_g") for k in keys)


def test_local_embed_none_and_absent():
    meta, _ = load_golden("vqvae_vctk_lg")
    m = _mirror(meta["kwargs"], local_embed_dim=None, decoder_conf=dict(meta["kwargs"]["decoder_conf"], in_channels=386))
    assert m.local_embed is None and not any(k.startswith("local_embed") for k in m.state_dict())
    m = _mirror(meta["kwargs"], num_local_embeds=None)
    assert not hasattr(m, "local_embed")


def test_rejected_configurations():
    meta, _ = load_golden("vqvae_yesno")
    with pytest.raises(NotImplementedError):
        _mirror(meta["kwargs"], decoder_type="HiFiGANGenerator", decoder_conf={"in_channels": 8})
    from parallelwavegan_b200 import losses, models, train_step
    from parallelwavegan_b200.capi import PwgbError

    m = _mirror(meta["kwargs"], in_channels=2)
    with pytest.raises(PwgbError, match="in_channels > 1"):
        train_step.GanTrainStep(m, None, {"mse": losses.MSELoss()}, None, None)
    with pytest.raises(PwgbError, match="mse"):
        train_step.GanTrainStep(_mirror(meta["kwargs"]), None, {}, None, None)
    assert isinstance(_mirror(meta["kwargs"]), models.VQVAE)


def test_collater_rejects_what_the_reference_rejects():
    from parallelwavegan_b200 import datasets

    for kw in (dict(use_local_condition=True), dict(use_global_condition=True)):
        with pytest.raises(AssertionError):
            datasets.Collater(use_aux_input=True, **kw)
        with pytest.raises((AssertionError, RuntimeError)):
            datasets.Collater(use_aux_input=False, use_duration=True, **kw)


def test_cpu_tensors_are_refused():
    from parallelwavegan_b200.capi import PwgbError

    meta, g = load_golden("vqvae_yesno")
    m = _mirror(meta["kwargs"])
    with pytest.raises(PwgbError, match="no CPU fallback"):
        m(g["x"])
    with pytest.raises(PwgbError):
        m.decode(g["indices"])
    with pytest.raises(PwgbError):
        m.codebook(g["z_e"])


def test_load_model_builds_vqvae(tmp_path):
    from parallelwavegan_b200 import models, utils

    meta, _ = load_golden("vqvae_vctk_lg")
    sd = vq_weights(meta, fold=False)
    path = tmp_path / "checkpoint.pkl"
    torch.save({"model": {"generator": sd}}, path)
    np.save(tmp_path / "stats.npy", np.zeros((2, 80), dtype=np.float32))  # present next to the checkpoint: not registered
    m = utils.load_model(str(path), config={"generator_type": "VQVAE", "generator_params": meta["kwargs"], "format": "npy"})
    assert type(m) is models.VQVAE and not hasattr(m, "mean") and not hasattr(m, "pqmf")
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
