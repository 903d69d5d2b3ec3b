"""Discrete-symbol StyleMelGAN generator without a GPU: the CPU oracle against the reference's golden outputs, the
mirror's module structure (state-dict names and shapes, weight-norm round trip, loading by config name), the
reference's failing inputs raising before any launch, and the decoder's host logic."""
import numpy as np
import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, golden_weights, load_golden, rel_l2
from oracle import ref_dsym_style, ref_ops

NAMES = ["dsym_style_small", "dsym_style_vctk"]


def _model(meta, **kw):
    from parallelwavegan_b200 import models

    return models.DiscreteSymbolStyleMelGANGenerator(**dict(meta["kwargs"], **kw))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    meta, g = load_golden(name)
    w, cfg = golden_effective_weights(meta), meta["kwargs"]
    with torch.no_grad():
        assert rel_l2(ref_dsym_style.dsym_style_generator(w, g["c"], g["z"], cfg), g["y"]) < ORACLE_TOL
        x0 = ref_dsym_style.noise_path(w, g["z"], cfg)
        assert rel_l2(x0, g["x0"]) < ORACLE_TOL
        x1, c1 = ref_ops.tade_res_block(w, "blocks.0", x0, ref_dsym_style.embed(w, g["c"], cfg), cfg["kernel_size"], cfg["dilation"],
                                        cfg["upsample_scales"][0], cfg["gated_function"])
        n = g["x1"].shape[-1]
        assert rel_l2(x1[..., :n], g["x1"]) < ORACLE_TOL and rel_l2(c1[..., :n], g["c1"]) < ORACLE_TOL
        f = int(np.prod(cfg["noise_upsample_scales"]))
        for k, T in enumerate(meta["inf_lengths"]):
            c, noise = g[f"inf{k}_c"], g[f"inf{k}_noise"]
            assert tuple(noise.shape) == (1, cfg["in_channels"], (T - 1) // f + 1)
            y = ref_dsym_style.dsym_style_inference(w, c, noise, cfg)
            assert tuple(y.shape) == (T * int(np.prod(cfg["upsample_scales"])), 1)
            assert rel_l2(y, g[f"inf{k}_y"]) < ORACLE_TOL
            if f"inf{k}_y_g" in g:
                cg = c.clone()
                cg[:, 1] = meta["g"]
                assert rel_l2(ref_dsym_style.dsym_style_inference(w, cg, noise, cfg), g[f"inf{k}_y_g"]) < ORACLE_TOL
    # one multiple of the noise length and one T the noise path is cropped to
    assert [T % f == 0 for T in meta["inf_lengths"]] == [True, False]


def test_recipe_shape():
    meta, g = load_golden("dsym_style_vctk")
    assert meta["n_params"] == 3560322
    assert [k for k, _ in meta["spec"][:4]] == ["emb.weight", "spk_emb.weight", "noise_upsample.0.bias", "noise_upsample.0.weight_g"]
    assert tuple(g["y"].shape) == (2, 1, 17920) and tuple(g["inf1_y"].shape) == (32000, 1)
    m = _model(meta)
    assert sum(p.numel() for p in m.parameters()) == 3560322
    assert (m.noise_upsample_factor, m.upsample_factor) == (56, 320)


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_matches_reference(name):
    meta, _ = load_golden(name)
    m = _model(meta)
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, list(s)) for k, s in meta["spec"]]
    m.load_state_dict(golden_weights(meta), strict=True)
    m.remove_weight_norm()
    folded = [(k[: -len("_v")] if k.endswith(".weight_v") else k, list(s)) for k, s in meta["spec"] if not k.endswith(".weight_g")]
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == folded
    m.apply_weight_norm()
    assert sorted(m.state_dict()) == sorted(k for k, _ in meta["spec"])
    # weight norm reaches the convs only: the embeddings keep a plain weight
    assert not any(k.startswith(("emb.", "spk_emb.")) and k.endswith(("_g", "_v")) for k, _ in meta["spec"])
    plain = _model(meta, use_weight_norm=False)
    plain.load_state_dict(golden_effective_weights(meta), strict=True)
    assert not hasattr(plain, "register_stats")


def test_reset_parameters_draws_every_conv_weight():
    meta, _ = load_golden("dsym_style_small")
    torch.manual_seed(0)
    m = _model(meta, use_weight_norm=False)
    convs = [(k, v) for k, v in m.state_dict().items() if k.endswith(".weight") and v.dim() == 3]
    assert len(convs) == 2 + 6 * 3 + 1
    w = torch.cat([v.reshape(-1) for _, v in convs])
    assert abs(float(w.std()) - 0.02) < 2e-3


def test_getattr_and_load_model(tmp_path):
    from parallelwavegan_b200 import models, utils

    meta, _ = load_golden("dsym_style_vctk")
    sd = golden_weights(meta)
    path = tmp_path / "checkpoint.pkl"
    torch.save({"model": {"generator": sd}}, path)
    gtype = "DiscreteSymbolStyleMelGANGenerator"
    m = utils.load_model(str(path), config={"generator_type": gtype, "generator_params": meta["kwargs"], "format": "npy"})
    assert type(m) is getattr(models, gtype)
    assert sorted(m.state_dict()) == sorted(sd) and all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())


def test_reference_failures_raise_before_any_launch():
    """concat_spk_emb=True constructs (the reference's state dict) and a T other than the noise length is accepted by the
    constructor; both fail at forward in the reference (verified there when the fixtures were made).  The mirror raises
    a RuntimeError with the reason from its host checks, before it reaches a kernel (which would refuse a CPU tensor)."""
    from parallelwavegan_b200.capi import PwgbError

    meta, g = load_golden("dsym_style_small")
    kw = meta["kwargs"]
    m = _model(meta, concat_spk_emb=True)
    assert m.blocks[0].tade1.aux_conv[0].in_channels == kw["aux_channels"] + kw["spk_emb_dim"]
    assert [(k, list(v.shape)) for k, v in m.state_dict().items() if k.startswith(("emb.", "spk_emb."))] == \
        [(k, list(s)) for k, s in meta["spec"] if k.startswith(("emb.", "spk_emb."))]
    with pytest.raises(PwgbError, match="concat_spk_emb"):
        m(g["c"], g["z"])
    with pytest.raises(PwgbError, match="concat_spk_emb"):
        m.inference(g["inf0_c"])
    m = _model(meta)
    with pytest.raises(PwgbError, match="noise path makes 12"):
        m(g["c"][:, :, :6], g["z"])
    with pytest.raises(PwgbError, match="noise path makes 6"):
        m(g["c"])  # the default z has one frame
    with pytest.raises(PwgbError, match=r"noise must be \(1, 16, 2\)"):
        m.inference(g["inf1_c"], noise=torch.zeros(1, 16, 1))
    with pytest.raises(AssertionError):
        m.inference(g["inf1_c"], normalize_before=True)


def test_decoder_host_logic():
    from parallelwavegan_b200 import decode, models
    from parallelwavegan_b200.capi import PwgbError

    meta, _ = load_golden("dsym_style_small")
    m = _model(meta)
    assert decode.decoder_kind(m) == "style_units"
    assert decode.decoder_kind(models.StyleMelGANGenerator()) == "style"
    with pytest.raises(PwgbError, match="InstanceNorm"):
        decode.Decoder(m, ragged=True)
    assert "InstanceNorm" in decode.ragged_refusal(m)
    with pytest.raises(PwgbError, match="CUDA"):
        decode.Decoder(m)

    def bare(kind, model):
        d = object.__new__(decode.Decoder)
        d.kind, d.model, d.rank, d.world, d.dev = kind, model, 0, 1, torch.device("cpu")
        return d

    units = [np.zeros((7, 2), np.int64), np.zeros((9, 2), np.int64)]
    with pytest.raises(PwgbError, match="normalize_before"):
        bare("style_units", m).decode(units, normalize_before=True)
    with pytest.raises(PwgbError, match="2 utterances"):
        bare("style_units", m).decode(units, speakers=[1])
    with pytest.raises(PwgbError, match=r"utterances \[1\] need one speaker id in \[0, 4\)"):
        bare("style_units", m).decode(units, speakers=[1, 4])
    with pytest.raises(PwgbError, match=r"\(T, 2\)"):
        bare("style_units", m).decode([np.zeros((7, 1), np.int64)])
    with pytest.raises(PwgbError, match="excitations are an input of the U-Net HiFi-GAN only"):
        bare("style_units", m).decode(units, excitations=[np.zeros(7 * 320), np.zeros(9 * 320)])
    with pytest.raises(PwgbError, match="draws its noise in inference"):
        bare("style_units", m).decode(units, noises={0: np.zeros((7 * 320, 1))})
    with pytest.raises(PwgbError, match="discrete-symbol StyleMelGAN only"):
        bare("mel2wav", models.HiFiGANGenerator(channels=32)).decode([np.zeros((3, 80), np.float32)], speakers=[0])
    # (T, 1) units with a speaker, or (T, 2) whose speaker column the speaker replaces
    assert tuple(decode._unit_rows(np.zeros((7, 1)), speakers=False).shape) == (7, 1)
    assert decode._speaker_list([np.int64(3), [2]], 2, [0, 1], 4) == {0: 3, 1: 2}
    assert decode._speaker_list(None, 2, [0, 1], 4) is None
