"""CPU restatement of the reference's discrete-symbol HiFi-GAN generators (TEST INFRASTRUCTURE), in the style of
``oracle.ref_ops.hifigan_generator``: effective (weight-norm folded) weights keyed like the reference ``state_dict()``
after ``remove_weight_norm()``, plain fp32 ATen ops, eval mode (dropout is the identity).

Citations are relative to ``/root/reference/``.  Parity status: pinned (see ``tests/test_discrete_symbol_cpu.py``).
"""
import torch
import torch.nn.functional as F

from oracle.ref_ops import hifigan_resblock


def embed(w, c, cfg):
    """c (B, 2, T) (symbol, speaker) or (B, 1, T) of any dtype -> (B, C, T) (hifigan.py:1005-1020): the indices are read
    as c.long(); the speaker is the first frame's, added to every frame."""
    c = c.long()
    e = F.embedding(c[:, 0], w["emb.weight"]).transpose(1, 2)
    if cfg.get("num_spk_embs", 128) > 0:
        e = e + F.embedding(c[:, 1, 0], w["spk_emb.weight"]).unsqueeze(2)
    return e


def body(w, c, cfg):
    """input_conv, per level LeakyReLU -> ConvTranspose1d(k, s, padding (k - s) // 2) and the MRF average, then
    LeakyReLU(0.01) -> output conv -> tanh (hifigan.py:938-986, 1022-1029)."""
    ks = cfg.get("kernel_size", 7)
    slope = cfg.get("nonlinear_activation_params", {"negative_slope": 0.1}).get("negative_slope", 0.1)
    nb = len(cfg["resblock_kernel_sizes"])
    c = F.conv1d(c, w["input_conv.weight"], w["input_conv.bias"], padding=(ks - 1) // 2)
    for i, (s, k) in enumerate(zip(cfg["upsample_scales"], cfg["upsample_kernel_sizes"])):
        c = F.conv_transpose1d(F.leaky_relu(c, slope), w[f"upsamples.{i}.1.weight"], w[f"upsamples.{i}.1.bias"], stride=s,
                               padding=(k - s) // 2)
        cs = 0.0
        for j in range(nb):
            cs = cs + hifigan_resblock(w, f"blocks.{i * nb + j}", c, cfg["resblock_kernel_sizes"][j], cfg["resblock_dilations"][j],
                                       cfg.get("use_additional_convs", True), slope)
        c = cs / nb
    c = F.conv1d(F.leaky_relu(c, 0.01), w["output_conv.1.weight"], w["output_conv.1.bias"], padding=(ks - 1) // 2)
    return torch.tanh(c)


def dsym_generator(w, c, cfg):
    """DiscreteSymbolHiFiGANGenerator.forward (hifigan.py:995-1031), add mode."""
    return body(w, embed(w, c, cfg), cfg)


def duration_predictor(w, e, cfg, prefix="duration_predictor"):
    """DurationPredictor._forward in log domain (layers/duration_predictor.py:71-77) on the channel-major (B, C, T)
    embedding: per layer Conv1d -> ReLU -> LayerNorm over channels (eps 1e-12, layers/layer_norm.py:34-40) -> Dropout
    (identity), then Linear(n_chans, 1)."""
    k = cfg.get("duration_kernel_size", 3)
    h = e
    for i in range(cfg.get("duration_layers", 2)):
        h = F.relu(F.conv1d(h, w[f"{prefix}.conv.{i}.0.weight"], w[f"{prefix}.conv.{i}.0.bias"], padding=(k - 1) // 2))
        h = F.layer_norm(h.transpose(1, 2), (h.shape[1],), w[f"{prefix}.conv.{i}.2.weight"], w[f"{prefix}.conv.{i}.2.bias"],
                         1e-12).transpose(1, 2)
    return F.linear(h.transpose(1, 2), w[f"{prefix}.linear.weight"], w[f"{prefix}.linear.bias"]).squeeze(-1)


def duration_round(x, offset=1.0):
    """DurationPredictor.inference (layers/duration_predictor.py:79-83): clamp(round(exp(x) - offset), min=0).long()."""
    return torch.clamp(torch.round(x.exp() - offset), min=0).long()


def length_regulate(e, ds):
    """LengthRegulator.forward (layers/length_regulator.py:71-98) on the channel-major (B, C, S) embedding -> (B, C, T*):
    when the whole batch sums to zero, rows summing to zero become all ones (in place on ``ds``); row b repeats symbol j
    ds[b, j] times; rows are zero-padded to the largest total."""
    if ds.sum() == 0:
        ds[ds.sum(dim=1).eq(0)] = 1
    rows = [torch.repeat_interleave(x, d, dim=1) for x, d in zip(e, ds)]
    t = max(r.shape[1] for r in rows)
    out = e.new_zeros(e.shape[0], e.shape[1], t)
    for b, r in enumerate(rows):
        out[b, :, : r.shape[1]] = r
    return out


def dsym_duration_forward(w, c, ds, cfg):
    """DiscreteSymbolDurationGenerator.forward (hifigan.py:1184-1223) -> (y, ds_out log-domain)."""
    e = embed(w, c, cfg)
    ds_out = duration_predictor(w, e, cfg)
    return body(w, length_regulate(e, ds), cfg), ds_out


def dsym_duration_synthesis(w, c, cfg):
    """DiscreteSymbolDurationGenerator.synthesis (hifigan.py:1250-1289) -> (y, int64 durations after the zero rule)."""
    e = embed(w, c, cfg)
    ds = duration_round(duration_predictor(w, e, cfg), cfg.get("duration_offset", 1.0))
    return body(w, length_regulate(e, ds), cfg), ds


def duration_loss(x, ds, offset=1.0):
    """DurationPredictorLoss (losses/duration_prediction_loss.py:34-52): MSELoss(mean) against log(ds + offset)."""
    return F.mse_loss(x, torch.log(ds.float() + offset))
