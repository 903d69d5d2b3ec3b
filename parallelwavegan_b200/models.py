"""Host-side mirror of ``parallel_wavegan.models``: same class names, constructor
kwargs, ``forward`` / ``inference`` signatures and ``state_dict()`` keys, so that
``getattr(models, config["generator_type"])(**config["generator_params"])``
(train.py:1364-1381, utils/utils.py:317-330) and reference checkpoints work
unchanged.  Forward passes run only on CUDA through ``libpwgb.so``.
"""
import logging

import numpy as np
import torch

from . import ops
from .capi import PwgbError
from .layers import HiFiGANResidualBlock as ResidualBlock
from .layers import CausalConv1d, CausalConvTranspose1d, ResidualStack, TADEResBlock, VQCodebook, activation_slope, effective_weight, pad_mode_of


def _read_stats(stats):
    assert stats.endswith(".h5") or stats.endswith(".npy")
    if stats.endswith(".h5"):
        import h5py  # optional dependency, as in the reference (utils/utils.py:83-117)

        with h5py.File(stats, "r") as f:
            mean = f["mean"][()].reshape(-1)
            scale = f["scale"][()].reshape(-1)
    else:
        mean = np.load(stats)[0].reshape(-1)
        scale = np.load(stats)[1].reshape(-1)
    return mean, scale


class _GeneratorBase(torch.nn.Module):
    def remove_weight_norm(self):
        def _remove_weight_norm(m):
            try:
                torch.nn.utils.remove_weight_norm(m)
            except ValueError:
                return

        self.apply(_remove_weight_norm)

    def register_stats(self, stats):
        mean, scale = _read_stats(stats)
        self.register_buffer("mean", torch.from_numpy(mean).float())
        self.register_buffer("scale", torch.from_numpy(scale).float())
        logging.info("Successfully registered stats as buffer.")

    def _prep_inference_input(self, c, normalize_before):
        if not isinstance(c, torch.Tensor):
            c = torch.tensor(c, dtype=torch.float).to(next(self.parameters()).device)
        if normalize_before:
            c = (c - self.mean) / self.scale
        return c.transpose(1, 0).unsqueeze(0).contiguous()


def _mrf_average(blocks, first, nb, h, differentiable, mask=None):
    """sum_j blocks[first + j](h) / nb: ScaledSumFn under autograd, else fused into each block's last conv.  ``mask``:
    the length mask of a ragged batch (inference only); the first block's last conv writes +0.0 outside each item's
    signal, which the later ones accumulate onto."""
    if differentiable:
        if mask is not None:
            raise PwgbError("per-item lengths are an inference feature (no autograd)")
        from .autograd import ScaledSumFn

        return ScaledSumFn.apply(1.0 / nb, *[blocks[first + j](h) for j in range(nb)])
    cs = torch.empty_like(h)
    for j in range(nb):
        if mask is None:
            blocks[first + j](h, out=cs, accumulate=j > 0, out_scale=1.0 / nb)
        else:
            blocks[first + j](h, out=cs, accumulate=j > 0, out_scale=1.0 / nb, mask=mask)
    return cs


def _length_mask(lengths, B, rate):
    """The pwgb_stream_ext mask of a ragged batch at ``rate`` samples per frame: item b is [0, lengths[b] * rate)."""
    if not (isinstance(lengths, torch.Tensor) and lengths.is_cuda and lengths.dtype == torch.int32 and lengths.dim() == 1
            and lengths.numel() == B and lengths.is_contiguous()):
        raise PwgbError(f"lengths must be {B} contiguous int32 frame counts on the device")
    return (torch.zeros_like(lengths), lengths, int(rate), 0)


def _masked(c, lengths, rate):
    """c with the samples past each item's length (``lengths`` frames at ``rate`` samples per frame) set to +0.0"""
    return c if lengths is None else ops.stream_mask(c, _length_mask(lengths, c.shape[0], rate))


def _hifigan_body(g, c, lengths=None):
    """The HiFi-GAN body after input_conv (hifigan.py:182-192, 1023-1029, 1215-1221, 1281-1287): per level LeakyReLU ->
    ConvTranspose1d (fused pre-activation) and the MRF average, then LeakyReLU(0.01) -> output conv -> tanh.  Shared by
    HiFiGANGenerator and the discrete-symbol generators; the conv-transpose padding is read from each module, which
    is where the two differ.  Inference runs the fused ResBlock pairs, autograd ScaledSumFn.

    ``lengths`` ((B,) int32 frame counts on the device, non-causal inference): a ragged batch whose input c is zero past
    each item's end.  Each conv-transpose output is masked with one pwgb_stream_mask (its kernels are the ones
    ``inference`` takes, and the mask pass is one read and write of a tensor that the MRF then reads 3 x 3 x 2 times),
    the MRF pairs mask in their epilogues, and the output conv needs none: nothing reads it.  Every sample of item b
    before lengths[b] * hop then equals ``forward`` of that item alone wherever both take the same kernels."""
    nb = g.num_blocks
    rate = 1
    for i in range(g.num_upsamples):
        up = g.upsamples[i][1]
        if g.use_causal_conv:
            c = up(c, pre_slope=g.slope)
        else:
            t_in = c.shape[-1]
            c = ops.conv_transpose1d(c, effective_weight(up), up.bias, stride=up.stride[0], padding=up.padding[0],
                                     output_padding=up.output_padding[0], pre_slope=g.slope)
        mask = None
        if lengths is not None:
            if c.shape[-1] != t_in * up.stride[0]:
                raise PwgbError(f"per-item lengths: upsampling level {i} maps {t_in} frames to {c.shape[-1]} samples, not "
                                f"{t_in} x {up.stride[0]}")
            rate *= up.stride[0]
            mask = _length_mask(lengths, c.shape[0], rate)
            ops.stream_mask(c, mask)
        c = _mrf_average(g.blocks, i * nb, nb, c, torch.is_grad_enabled() and (c.requires_grad or next(g.parameters()).requires_grad),
                         mask)
    oc = g.output_conv[1]
    if g.use_causal_conv:
        return oc(c, pre_slope=0.01, post_act="tanh")
    return ops.conv1d(c, effective_weight(oc), oc.bias, padding=(g.kernel_size - 1) // 2, pre_slope=0.01, post_act="tanh")


class HiFiGANGenerator(_GeneratorBase):
    """models/hifigan.py:23-267."""

    def __init__(
        self,
        in_channels=80,
        out_channels=1,
        channels=512,
        kernel_size=7,
        upsample_scales=(8, 8, 2, 2),
        upsample_kernel_sizes=(16, 16, 4, 4),
        resblock_kernel_sizes=(3, 7, 11),
        resblock_dilations=[(1, 3, 5), (1, 3, 5), (1, 3, 5)],
        use_additional_convs=True,
        bias=True,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.1},
        use_causal_conv=False,
        use_weight_norm=True,
    ):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernel size must be odd number."
        assert len(upsample_scales) == len(upsample_kernel_sizes)
        assert len(resblock_dilations) == len(resblock_kernel_sizes)
        self.num_upsamples = len(upsample_kernel_sizes)
        self.num_blocks = len(resblock_kernel_sizes)
        self.use_causal_conv = use_causal_conv
        self.kernel_size = kernel_size
        self.upsample_scales = tuple(upsample_scales)
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        act = getattr(torch.nn, nonlinear_activation)
        if use_causal_conv:
            self.input_conv = CausalConv1d(in_channels, channels, kernel_size, bias=bias)
        else:
            self.input_conv = torch.nn.Conv1d(in_channels, channels, kernel_size, bias=bias, padding=(kernel_size - 1) // 2)
        self.upsamples = torch.nn.ModuleList()
        self.blocks = torch.nn.ModuleList()
        for i in range(len(upsample_kernel_sizes)):
            assert upsample_kernel_sizes[i] == 2 * upsample_scales[i]
            s = upsample_scales[i]
            if use_causal_conv:
                up = CausalConvTranspose1d(channels // (2**i), channels // (2 ** (i + 1)), upsample_kernel_sizes[i], s, bias=bias)
            else:
                up = torch.nn.ConvTranspose1d(
                    channels // (2**i), channels // (2 ** (i + 1)), upsample_kernel_sizes[i], s,
                    padding=s // 2 + s % 2, output_padding=s % 2, bias=bias,
                )
            self.upsamples += [torch.nn.Sequential(act(**nonlinear_activation_params), up)]
            for j in range(len(resblock_kernel_sizes)):
                self.blocks += [
                    ResidualBlock(
                        kernel_size=resblock_kernel_sizes[j],
                        channels=channels // (2 ** (i + 1)),
                        dilations=resblock_dilations[j],
                        bias=bias,
                        use_additional_convs=use_additional_convs,
                        nonlinear_activation=nonlinear_activation,
                        nonlinear_activation_params=nonlinear_activation_params,
                        use_causal_conv=use_causal_conv,
                    )
                ]
        self.output_conv = torch.nn.Sequential(
            torch.nn.LeakyReLU(),  # default slope 0.01 (hifigan.py:139-142)
            CausalConv1d(channels // (2 ** (i + 1)), out_channels, kernel_size, bias=bias)
            if use_causal_conv
            else torch.nn.Conv1d(channels // (2 ** (i + 1)), out_channels, kernel_size, bias=bias, padding=(kernel_size - 1) // 2),
            torch.nn.Tanh(),
        )
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    def forward(self, c, lengths=None):
        """(B, in_channels, T) -> (B, out_channels, T * prod(upsample_scales))  (hifigan.py:173-192).

        ``lengths``: (B,) int32 frame counts on the device, for a batch of utterances of different lengths padded with
        zero frames (inference).  Item b's first lengths[b] * hop samples are then the forward of its first lengths[b]
        frames alone (see _hifigan_body); the rest is padding.  A causal generator needs no mask: its outputs never
        read later frames, so it ignores ``lengths``."""
        ic = self.input_conv
        if self.use_causal_conv:
            return _hifigan_body(self, ic(c))
        c = ops.conv1d(c, effective_weight(ic), ic.bias, padding=(self.kernel_size - 1) // 2)
        return _hifigan_body(self, _masked(c, lengths, 1), lengths)

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.01)

        self.apply(_reset_parameters)

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def inference(self, c, normalize_before=False):
        """(T, in_channels) -> (T * prod(upsample_scales), out_channels)  (hifigan.py:251-267)."""
        c = self.forward(self._prep_inference_input(c, normalize_before))
        return c.squeeze(0).transpose(1, 0)


class DiscreteSymbolHiFiGANGenerator(torch.nn.Module):
    """models/hifigan.py:867-1091: HiFi-GAN over discrete units (HuBERT codes).  The symbol embedding (+ the speaker
    embedding of each item's first frame) is written channel-major by one embed launch (pwgb_symbol_embed_forward),
    reading the index tensor in place; the body is HiFiGANGenerator's (``_hifigan_body``).  The upsampling
    ConvTranspose1d uses padding (k - s) // 2 and no output_padding (hifigan.py:953-959).  There is no
    ``register_stats``, as in the reference."""

    def __init__(
        self,
        in_channels=512,
        out_channels=1,
        channels=512,
        num_embs=100,
        num_spk_embs=128,
        spk_emb_dim=128,
        concat_spk_emb=False,
        kernel_size=7,
        upsample_scales=(8, 8, 2, 2),
        upsample_kernel_sizes=(16, 16, 4, 4),
        resblock_kernel_sizes=(3, 7, 11),
        resblock_dilations=[(1, 3, 5), (1, 3, 5), (1, 3, 5)],
        use_additional_convs=True,
        bias=True,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.1},
        use_weight_norm=True,
    ):
        super().__init__()
        self.num_spk_embs = num_spk_embs
        self.emb = torch.nn.Embedding(num_embeddings=num_embs, embedding_dim=in_channels)
        if self.num_spk_embs > 0:
            self.spk_emb = torch.nn.Embedding(num_embeddings=num_spk_embs, embedding_dim=spk_emb_dim)
            self.concat_spk_emb = concat_spk_emb
            if not concat_spk_emb:
                assert in_channels == spk_emb_dim
            else:
                in_channels = in_channels + spk_emb_dim
        assert kernel_size % 2 == 1, "Kernal size must be odd number."
        assert len(upsample_scales) == len(upsample_kernel_sizes)
        assert len(resblock_dilations) == len(resblock_kernel_sizes)
        self.num_upsamples = len(upsample_kernel_sizes)
        self.num_blocks = len(resblock_kernel_sizes)
        self.use_causal_conv = False
        self.kernel_size = kernel_size
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        act = getattr(torch.nn, nonlinear_activation)
        # input / upsampling / output convs always have a bias; ``bias`` reaches the residual blocks only (hifigan.py:938-986)
        self.input_conv = torch.nn.Conv1d(in_channels, channels, kernel_size, 1, padding=(kernel_size - 1) // 2)
        self.upsamples = torch.nn.ModuleList()
        self.blocks = torch.nn.ModuleList()
        for i in range(len(upsample_kernel_sizes)):
            self.upsamples += [
                torch.nn.Sequential(
                    act(**nonlinear_activation_params),
                    torch.nn.ConvTranspose1d(channels // (2**i), channels // (2 ** (i + 1)), upsample_kernel_sizes[i], upsample_scales[i],
                                             padding=(upsample_kernel_sizes[i] - upsample_scales[i]) // 2),
                )
            ]
            for j in range(len(resblock_kernel_sizes)):
                self.blocks += [
                    ResidualBlock(
                        kernel_size=resblock_kernel_sizes[j],
                        channels=channels // (2 ** (i + 1)),
                        dilations=resblock_dilations[j],
                        bias=bias,
                        use_additional_convs=use_additional_convs,
                        nonlinear_activation=nonlinear_activation,
                        nonlinear_activation_params=nonlinear_activation_params,
                    )
                ]
        self.output_conv = torch.nn.Sequential(
            torch.nn.LeakyReLU(),  # default slope 0.01 (hifigan.py:974-986)
            torch.nn.Conv1d(channels // (2 ** (i + 1)), out_channels, kernel_size, 1, padding=(kernel_size - 1) // 2),
            torch.nn.Tanh(),
        )
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    remove_weight_norm = _GeneratorBase.remove_weight_norm
    reset_parameters = HiFiGANGenerator.reset_parameters
    apply_weight_norm = HiFiGANGenerator.apply_weight_norm

    def _check_input(self, c):
        if self.num_spk_embs > 0:
            assert c.size(1) == 2
            if self.concat_spk_emb:
                # hifigan.py:1015-1017 concatenates the speaker embedding along time, so input_conv, built for
                # in_channels + spk_emb_dim, receives in_channels: the reference fails there; so does the mirror
                raise PwgbError(f"concat_spk_emb=True: input_conv expects {self.input_conv.in_channels} channels, the embedding "
                                f"has {self.emb.embedding_dim} (the reference concatenates the speaker embedding along time)")
        else:
            assert c.size(1) == 1

    def _embed(self, c, ds=None, t_out=None, symbol_level=False):
        """(B, 1 or 2, S) symbol (, speaker) indices of any dtype -> channel-major embedding (see ops.symbol_embed)."""
        self._check_input(c)
        spk = self.spk_emb.weight if self.num_spk_embs > 0 else None
        return ops.symbol_embed(c, self.emb.weight, spk, ds=ds, t_out=t_out, symbol_level=symbol_level)

    def _body(self, c, lengths=None):
        ic = self.input_conv
        c = ops.conv1d(_masked(c, lengths, 1), effective_weight(ic), ic.bias, padding=(self.kernel_size - 1) // 2)
        return _hifigan_body(self, _masked(c, lengths, 1), lengths)

    def forward(self, c, lengths=None):
        """c (B, 2, T) (symbol, speaker id) or (B, 1, T) -> (B, out_channels, T * prod(upsample_scales))  (hifigan.py:995-1031).

        ``lengths``: (B,) int32 frame counts on the device (inference), as in HiFiGANGenerator.forward; the embedding of
        the indices past an item's end (any symbol) is masked to zero before input_conv, and each item's speaker is its
        own first frame's."""
        return self._body(self._embed(c), lengths)

    def _prep_symbols(self, c, g):
        """inference input plumbing (hifigan.py:1082-1090): (T, 2) or (T, 1) -> (1, K, T) view."""
        if not isinstance(c, torch.Tensor):
            c = torch.tensor(c, dtype=torch.long).to(next(self.parameters()).device)
        if g is not None:
            c = c[:, 0:1]
            c = torch.cat([c, c.new_zeros(*c.size()).fill_(g).to(c.device)], dim=1)
        if self.num_spk_embs <= 0:
            c = c[:, 0:1]
        return c.transpose(1, 0).unsqueeze(0)

    def inference(self, c, g=None, normalize_before=False):
        """(T, 2) or (T, 1) indices [, speaker id g] -> (T * prod(upsample_scales), out_channels)  (hifigan.py:1072-1091)."""
        assert not normalize_before, "No statistics are used."
        c = self.forward(self._prep_symbols(c, g))
        return c.squeeze(0).transpose(1, 0)


class DiscreteSymbolDurationGenerator(DiscreteSymbolHiFiGANGenerator):
    """models/hifigan.py:1094-1289: the discrete-symbol generator with a FastSpeech duration predictor and a length
    regulator.  ``forward(c, ds)`` regulates by the given durations, ``synthesis`` by the predicted ones.  The embedding
    is gathered twice from the table by one autograd Function: per symbol for the predictor and length-regulated for
    input_conv.  Sizing the regulated tensor reads the B row totals on the host (one small device-to-host copy per
    forward with durations, where the reference synchronises too).  The duration predictor is built after weight
    norm, so its convs are plain (hifigan.py:1170-1182)."""

    def __init__(
        self,
        in_channels=512,
        out_channels=1,
        channels=512,
        num_embs=100,
        num_spk_embs=128,
        spk_emb_dim=128,
        concat_spk_emb=False,
        duration_layers=2,
        duration_chans=384,
        duration_kernel_size=3,
        duration_offset=1.0,
        duration_dropout_rate=0.5,
        kernel_size=7,
        upsample_scales=(8, 8, 2, 2),
        upsample_kernel_sizes=(16, 16, 4, 4),
        resblock_kernel_sizes=(3, 7, 11),
        resblock_dilations=[(1, 3, 5), (1, 3, 5), (1, 3, 5)],
        use_additional_convs=True,
        bias=True,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.1},
        use_weight_norm=True,
    ):
        from .layers import DurationPredictor, LengthRegulator

        super().__init__(
            in_channels=in_channels, out_channels=out_channels, channels=channels, num_embs=num_embs + 1,  # + the padding symbol
            num_spk_embs=num_spk_embs, spk_emb_dim=spk_emb_dim, concat_spk_emb=concat_spk_emb, kernel_size=kernel_size,
            upsample_scales=upsample_scales, upsample_kernel_sizes=upsample_kernel_sizes, resblock_kernel_sizes=resblock_kernel_sizes,
            resblock_dilations=resblock_dilations, use_additional_convs=use_additional_convs, bias=bias,
            nonlinear_activation=nonlinear_activation, nonlinear_activation_params=nonlinear_activation_params,
            use_weight_norm=use_weight_norm,
        )
        if self.num_spk_embs > 0:
            # built for in_channels + spk_emb_dim inputs but fed in_channels: forward raises, as in the reference
            in_channels = in_channels + spk_emb_dim
        self.duration_predictor = DurationPredictor(in_channels, n_layers=duration_layers, n_chans=duration_chans,
                                                    kernel_size=duration_kernel_size, dropout_rate=duration_dropout_rate,
                                                    offset=duration_offset)
        self.length_regulator = LengthRegulator()

    def _check_input(self, c):
        super()._check_input(c)
        if self.duration_predictor.conv[0][0].in_channels != self.emb.embedding_dim:
            # num_spk_embs > 0: the predictor is built for in_channels + spk_emb_dim inputs and receives in_channels
            # (hifigan.py:1170-1180, 1211); the reference fails at its first conv, the mirror before any launch
            raise PwgbError(f"duration predictor expects {self.duration_predictor.conv[0][0].in_channels} channels, the embedding "
                            f"has {self.emb.embedding_dim} (the reference builds it for in_channels + spk_emb_dim)")

    def forward(self, c, ds):
        """c (B, 2 or 1, S), ds (B, S) int64 -> (y (B, out_channels, max_b sum(ds[b]) * prod(upsample_scales)), ds_out (B, S)
        log-domain predicted durations)  (hifigan.py:1184-1223).  ``ds`` gets the length regulator's all-zero rule in
        place, as in the reference."""
        self._check_input(c)
        _, totals = ops.duration_round(None, ds=ds)
        e, e_sym = self._embed(c, ds=ds, t_out=ops.regulated_length(totals), symbol_level=True)
        ds_out = self.duration_predictor(e_sym.transpose(1, 2))
        return self._body(e), ds_out

    def synthesis(self, c):
        """c (B, 2 or 1, S) -> (y, ds_out (B, S) int64 predicted durations after the all-zero rule)  (hifigan.py:1250-1289)."""
        e_sym = self._embed(c)
        x = self.duration_predictor._log_durations(e_sym.transpose(1, 2), None)
        ds, totals = ops.duration_round(x, self.duration_predictor.offset)  # rounding and the regulator's rule: one launch
        e = self._embed(c, ds=ds, t_out=ops.regulated_length(totals))
        return self._body(e), ds

    def inference(self, c, g=None, ds=None, normalize_before=False):
        """(T, 2) or (T, 1) indices [, speaker id g] [, durations ds (T,)] -> (sum(ds) * prod(upsample_scales), out_channels)
        (hifigan.py:1225-1248)."""
        assert not normalize_before, "No statistics are used."
        c = self._prep_symbols(c, g)
        if ds is None:
            y, _ = self.synthesis(c)
        else:
            y, _ = self.forward(c, ds.unsqueeze(0))
        return y.squeeze(0).transpose(1, 0)


class UHiFiGANGenerator(_GeneratorBase):
    """models/uhifigan.py:19-343: a U-Net over the excitation signal.  The encoder (input conv, then per level the MRF
    and a strided conv) keeps each level's output; the decoder starts from the mel features (hidden_conv) and on every
    level runs LeakyReLU -> ConvTranspose1d over cat(decoder state, encoder output), then the MRF.  The concatenation
    is never materialised: the conv-transpose reads its input channels from the two tensors."""

    def __init__(
        self,
        in_channels=80,
        out_channels=1,
        channels=512,
        kernel_size=7,
        downsample_scales=(8, 8, 2, 2),
        downsample_kernel_sizes=(16, 16, 4, 4),
        upsample_scales=(8, 8, 2, 2),
        upsample_kernel_sizes=(16, 16, 4, 4),
        resblock_kernel_sizes=(3, 7, 11),
        resblock_dilations=[(1, 3, 5), (1, 3, 5), (1, 3, 5)],
        dropout=0.3,
        use_additional_convs=True,
        bias=True,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.1},
        use_causal_conv=False,
        use_weight_norm=True,
    ):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernel size must be odd number."
        assert len(upsample_scales) == len(upsample_kernel_sizes)
        assert len(resblock_dilations) == len(resblock_kernel_sizes)
        self.num_upsamples = len(upsample_kernel_sizes)
        self.num_blocks = len(resblock_kernel_sizes)
        self.use_causal_conv = use_causal_conv
        self.kernel_size = kernel_size
        self.downsample_scales = tuple(downsample_scales)
        self.upsample_scales = tuple(upsample_scales)
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        act = getattr(torch.nn, nonlinear_activation)
        self.downsamples = torch.nn.ModuleList()
        self.downsamples_mrf = torch.nn.ModuleList()
        self.upsamples = torch.nn.ModuleList()
        self.upsamples_mrf = torch.nn.ModuleList()
        # the reference passes padding= to CausalConv1d, which has no such argument: use_causal_conv=True raises
        # TypeError here as it does there (uhifigan.py:91-101)
        conv = CausalConv1d if use_causal_conv else torch.nn.Conv1d
        self.input_conv = torch.nn.Sequential(
            conv(out_channels, channels, kernel_size=kernel_size, bias=bias, padding=(kernel_size - 1) // 2),
            act(**nonlinear_activation_params),
            torch.nn.Dropout(dropout),
        )
        for i in range(len(downsample_scales)):
            for j in range(len(resblock_kernel_sizes)):
                self.downsamples_mrf += [
                    ResidualBlock(
                        kernel_size=resblock_kernel_sizes[j],
                        channels=channels,
                        dilations=resblock_dilations[j],
                        bias=bias,
                        use_additional_convs=use_additional_convs,
                        nonlinear_activation=nonlinear_activation,
                        nonlinear_activation_params=nonlinear_activation_params,
                        use_causal_conv=use_causal_conv,
                    )
                ]
            s = downsample_scales[i]
            self.downsamples += [
                torch.nn.Sequential(
                    torch.nn.Conv1d(channels, channels * 2, kernel_size=downsample_kernel_sizes[i], stride=s, bias=bias,
                                    padding=s // 2 + s % 2),
                    act(**nonlinear_activation_params),
                    torch.nn.Dropout(dropout),
                )
            ]
            channels = channels * 2
        self.hidden_conv = torch.nn.Conv1d(in_channels, channels, kernel_size=kernel_size, bias=bias, padding=(kernel_size - 1) // 2)
        for i in range(len(upsample_kernel_sizes)):
            s = upsample_scales[i]
            self.upsamples += [
                torch.nn.Sequential(
                    act(**nonlinear_activation_params),
                    torch.nn.ConvTranspose1d(channels * 2, channels // 2, upsample_kernel_sizes[i], s, padding=s // 2 + s % 2,
                                             output_padding=s % 2, bias=bias),
                )
            ]
            for j in range(len(resblock_kernel_sizes)):
                self.upsamples_mrf += [
                    ResidualBlock(
                        kernel_size=resblock_kernel_sizes[j],
                        channels=channels // 2,
                        dilations=resblock_dilations[j],
                        bias=bias,
                        use_additional_convs=use_additional_convs,
                        nonlinear_activation=nonlinear_activation,
                        nonlinear_activation_params=nonlinear_activation_params,
                        use_causal_conv=use_causal_conv,
                    )
                ]
            channels = channels // 2
        self.output_conv = torch.nn.Sequential(
            torch.nn.LeakyReLU(),  # default slope 0.01 (uhifigan.py:222-235)
            torch.nn.Conv1d(channels, out_channels, kernel_size, bias=bias, padding=(kernel_size - 1) // 2),
            torch.nn.Tanh(),
        )
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    def forward(self, c=None, f0=None, excitation=None):
        """c (B, in_channels, T'), excitation (B, 1, T' * hop) -> (B, out_channels, T' * hop)  (uhifigan.py:262-301).
        ``f0`` is accepted and unused, as in the reference."""
        pad = (self.kernel_size - 1) // 2
        nb = self.num_blocks
        slope = self.slope
        grad = torch.is_grad_enabled() and next(self.parameters()).requires_grad  # autograd: ScaledSumFn for the MRF average
        ic = self.input_conv[0]
        h = ops.conv1d(excitation, effective_weight(ic), ic.bias, padding=pad, post_act="lrelu", post_slope=slope)
        h = ops.dropout(h, self.input_conv[2].p, self.training)
        skips = []
        for i, ds in enumerate(self.downsamples):
            h = _mrf_average(self.downsamples_mrf, i * nb, nb, h, grad or h.requires_grad)
            s = self.downsample_scales[i]
            h = ops.conv1d(h, effective_weight(ds[0]), ds[0].bias, stride=s, padding=s // 2 + s % 2, post_act="lrelu",
                           post_slope=slope)
            h = ops.dropout(h, ds[2].p, self.training)
            skips.append(h)
        hc = self.hidden_conv
        h = ops.conv1d(c, effective_weight(hc), hc.bias, padding=pad)
        for i in range(self.num_upsamples):
            up = self.upsamples[i][1]
            s = self.upsample_scales[i]
            h = ops.conv_transpose1d_cat(h, skips[-1 - i], effective_weight(up), up.bias, stride=s, padding=s // 2 + s % 2,
                                         output_padding=s % 2, pre_slope=slope)
            h = _mrf_average(self.upsamples_mrf, i * nb, nb, h, grad or h.requires_grad)
        oc = self.output_conv[1]
        return ops.conv1d(h, effective_weight(oc), oc.bias, padding=pad, pre_slope=0.01, post_act="tanh")

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.01)

        self.apply(_reset_parameters)

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def inference(self, excitation=None, f0=None, c=None, normalize_before=False):
        """excitation (T' * hop,) or (T', hop), c (T', in_channels) -> (T' * hop, out_channels)  (uhifigan.py:317-343).
        ``normalize_before`` is ignored, as in the reference."""
        dev = next(self.parameters()).device
        if c is not None and not isinstance(c, torch.Tensor):
            c = torch.tensor(c, dtype=torch.float).to(dev)
        if excitation is not None and not isinstance(excitation, torch.Tensor):
            excitation = torch.tensor(excitation, dtype=torch.float).to(dev)
        if f0 is not None and not isinstance(f0, torch.Tensor):
            f0 = torch.tensor(f0, dtype=torch.float).to(dev)
        y = self.forward(
            c.transpose(1, 0).unsqueeze(0).contiguous(),
            f0.unsqueeze(1).transpose(1, 0).unsqueeze(0) if f0 is not None else None,
            excitation.reshape(1, 1, -1).contiguous(),
        )
        return y.squeeze(0).transpose(1, 0)


class MelGANGenerator(_GeneratorBase):
    """models/melgan.py:17-257 (also the multi-band generator with out_channels=4)."""

    def __init__(
        self,
        in_channels=80,
        out_channels=1,
        kernel_size=7,
        channels=512,
        bias=True,
        upsample_scales=[8, 8, 2, 2],
        stack_kernel_size=3,
        stacks=3,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.2},
        pad="ReflectionPad1d",
        pad_params={},
        use_final_nonlinear_activation=True,
        use_weight_norm=True,
        use_causal_conv=False,
    ):
        super().__init__()
        assert channels >= np.prod(upsample_scales)
        assert channels % (2 ** len(upsample_scales)) == 0
        if not use_causal_conv:
            assert (kernel_size - 1) % 2 == 0, "Not support even number kernel size."
        self.kernel_size = kernel_size
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        self.pad_mode = pad_mode_of(pad, pad_params)
        self.use_final_nonlinear_activation = use_final_nonlinear_activation
        act = getattr(torch.nn, nonlinear_activation)
        if use_causal_conv:
            layers = [CausalConv1d(in_channels, channels, kernel_size, bias=bias, pad=pad, pad_params=pad_params)]
        else:
            layers = [getattr(torch.nn, pad)((kernel_size - 1) // 2, **pad_params), torch.nn.Conv1d(in_channels, channels, kernel_size, bias=bias)]
        for i, s in enumerate(upsample_scales):
            layers += [act(**nonlinear_activation_params)]
            if use_causal_conv:
                layers += [CausalConvTranspose1d(channels // (2**i), channels // (2 ** (i + 1)), s * 2, stride=s, bias=bias)]
            else:
                layers += [
                    torch.nn.ConvTranspose1d(channels // (2**i), channels // (2 ** (i + 1)), s * 2, stride=s,
                                             padding=s // 2 + s % 2, output_padding=s % 2, bias=bias)
                ]
            for j in range(stacks):
                layers += [
                    ResidualStack(
                        kernel_size=stack_kernel_size,
                        channels=channels // (2 ** (i + 1)),
                        dilation=stack_kernel_size**j,
                        bias=bias,
                        nonlinear_activation=nonlinear_activation,
                        nonlinear_activation_params=nonlinear_activation_params,
                        pad=pad,
                        pad_params=pad_params,
                        use_causal_conv=use_causal_conv,
                    )
                ]
        layers += [act(**nonlinear_activation_params)]
        if use_causal_conv:
            layers += [CausalConv1d(channels // (2 ** (i + 1)), out_channels, kernel_size, bias=bias, pad=pad, pad_params=pad_params)]
        else:
            layers += [getattr(torch.nn, pad)((kernel_size - 1) // 2, **pad_params), torch.nn.Conv1d(channels // (2 ** (i + 1)), out_channels, kernel_size, bias=bias)]
        if use_final_nonlinear_activation:
            layers += [torch.nn.Tanh()]
        self.melgan = torch.nn.Sequential(*layers)
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()
        self.pqmf = None

    def forward(self, c, lengths=None):
        """(B, in_channels, T) -> (B, out_channels, T * prod(upsample_scales))  (melgan.py:168-178).

        ``lengths`` ((B,) int32 frame counts on the device, centred inference): a ragged batch.  Every conv keeps each
        item +0.0 past its own end and pads it at its own end -- the reflect-padded input, stack and output convs reflect
        there (pwgb_conv1d_ragged_forward) -- and each conv-transpose output is masked with one pwgb_stream_mask.  Every
        sample of item b before lengths[b] * hop then equals ``forward`` of that item alone wherever both take the same
        kernels (DESIGN.md §3.16)."""
        pad = (self.kernel_size - 1) // 2
        mods = list(self.melgan)
        n = len(mods)
        pre = 1.0  # slope of a pending activation, fused into the next conv's loader
        idx = 0
        mask, rate = None, 1
        if lengths is not None:
            if isinstance(mods[0], CausalConv1d):
                raise PwgbError("MelGANGenerator: per-item lengths serve the centred generator (use_causal_conv=False)")
            mask = _length_mask(lengths, c.shape[0], rate)
        kw = {} if mask is None else {"mask": mask}
        while idx < n:
            m = mods[idx]
            if isinstance(m, CausalConvTranspose1d):
                c = m(c, pre_slope=pre)
                pre = 1.0
            elif isinstance(m, CausalConv1d):
                final = idx >= n - 2
                c = m(c, pre_slope=pre, post_act="tanh" if (final and self.use_final_nonlinear_activation) else None)
                pre = 1.0
            elif isinstance(m, torch.nn.ConvTranspose1d):
                s = m.stride[0]
                c = ops.conv_transpose1d(c, effective_weight(m), m.bias, stride=s, padding=m.padding[0],
                                         output_padding=m.output_padding[0], pre_slope=pre)
                pre = 1.0
                if mask is not None:
                    rate *= s
                    mask = _length_mask(lengths, c.shape[0], rate)
                    kw = {"mask": mask}
                    ops.stream_mask(c, mask)
            elif isinstance(m, torch.nn.Conv1d):
                final = idx >= n - 2
                c = ops.conv1d(c, effective_weight(m), m.bias, padding=pad, pad_mode=self.pad_mode, pre_slope=pre,
                               post_act="tanh" if (final and self.use_final_nonlinear_activation) else None, **kw)
                pre = 1.0
            elif isinstance(m, ResidualStack):
                c = m(c, **kw)
            elif isinstance(m, (torch.nn.LeakyReLU, torch.nn.ReLU)):
                pre = self.slope
            # padding modules and the final Tanh are fused into the neighbouring conv
            idx += 1
        return c

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.02)

        self.apply(_reset_parameters)

    def inference(self, c, normalize_before=False):
        """(T, in_channels) -> (T * prod(upsample_scales) [* subbands], 1)  (melgan.py:239-257)."""
        c = self.forward(self._prep_inference_input(c, normalize_before))
        if self.pqmf is not None:
            c = self.pqmf.synthesis(c)
        return c.squeeze(0).transpose(1, 0)


class StyleMelGANGenerator(_GeneratorBase):
    """models/style_melgan.py:22-270 (forward / inference; trainable: the TADE glue has adjoint kernels)."""

    def __init__(
        self,
        in_channels=128,
        aux_channels=80,
        channels=64,
        out_channels=1,
        kernel_size=9,
        dilation=2,
        bias=True,
        noise_upsample_scales=[11, 2, 2, 2],
        noise_upsample_activation="LeakyReLU",
        noise_upsample_activation_params={"negative_slope": 0.2},
        upsample_scales=[2, 2, 2, 2, 2, 2, 2, 2, 1],
        upsample_mode="nearest",
        gated_function="softmax",
        use_weight_norm=True,
    ):
        super().__init__()
        self.in_channels = in_channels
        self._build(aux_channels, channels, out_channels, kernel_size, dilation, bias, noise_upsample_scales, noise_upsample_activation,
                    noise_upsample_activation_params, upsample_scales, upsample_mode, gated_function)
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    def _build(self, aux_channels, channels, out_channels, kernel_size, dilation, bias, noise_upsample_scales, noise_upsample_activation,
               noise_upsample_activation_params, upsample_scales, upsample_mode, gated_function):
        """noise_upsample, blocks and output_conv (style_melgan.py:62-131), registered in the reference's order."""
        self.noise_slope = activation_slope(noise_upsample_activation, noise_upsample_activation_params)
        noise_upsample = []
        in_chs = self.in_channels
        for s in noise_upsample_scales:
            noise_upsample += [torch.nn.ConvTranspose1d(in_chs, channels, s * 2, stride=s, padding=s // 2 + s % 2,
                                                        output_padding=s % 2, bias=bias)]
            noise_upsample += [getattr(torch.nn, noise_upsample_activation)(**noise_upsample_activation_params)]
            in_chs = channels
        self.noise_upsample = torch.nn.Sequential(*noise_upsample)
        self.noise_upsample_factor = int(np.prod(noise_upsample_scales))
        self.blocks = torch.nn.ModuleList()
        aux_chs = aux_channels
        for s in upsample_scales:
            self.blocks += [TADEResBlock(in_channels=channels, aux_channels=aux_chs, kernel_size=kernel_size, dilation=dilation,
                                         bias=bias, upsample_factor=s, upsample_mode=upsample_mode, gated_function=gated_function)]
            aux_chs = channels
        self.upsample_factor = int(np.prod(upsample_scales))
        self.kernel_size = kernel_size
        self.output_conv = torch.nn.Sequential(
            torch.nn.Conv1d(channels, out_channels, kernel_size, 1, bias=bias, padding=(kernel_size - 1) // 2),
            torch.nn.Tanh(),
        )

    def _noise_path(self, z):
        """noise_upsample (style_melgan.py:76-98): every LeakyReLU but the last is fused into the next
        transposed conv's loader; the last one is applied explicitly (the block needs it as the residual)."""
        x, pre = z, 1.0
        for m in self.noise_upsample:
            if isinstance(m, torch.nn.ConvTranspose1d):
                x = ops.conv_transpose1d(x, effective_weight(m), m.bias, stride=m.stride[0], padding=m.padding[0],
                                         output_padding=m.output_padding[0], pre_slope=pre)
                pre = self.noise_slope
        return ops.leaky_relu(x, self.noise_slope, inplace=True)

    def _body(self, x, c):
        """The TADE blocks and the output conv -> tanh on the noise path's x and the conditioning c (style_melgan.py:155-159)."""
        for block in self.blocks:
            x, c = block(x, c)
        oc = self.output_conv[0]
        return ops.conv1d(x, effective_weight(oc), oc.bias, padding=(self.kernel_size - 1) // 2, post_act="tanh")

    def forward(self, c, z=None):
        """(B, aux_channels, T) [, (B, in_channels, T_z)] -> (B, out_channels, T * prod(upsample_scales))  (style_melgan.py:140-160)."""
        if z is None:
            z = torch.randn(c.size(0), self.in_channels, 1).to(device=c.device, dtype=c.dtype)
        return self._body(self._noise_path(z), c)

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.02)

        self.apply(_reset_parameters)

    def inference(self, c, normalize_before=False, noise=None):
        """(T, aux_channels) -> (T * prod(upsample_scales), out_channels)  (style_melgan.py:226-262); ``noise``
        (1, in_channels, ceil(T / noise_upsample_factor)) may be passed for reproducibility."""
        c = self._prep_inference_input(c, normalize_before)
        n_frames = (c.size(2) - 1) // self.noise_upsample_factor + 1
        if noise is None:
            noise = torch.randn(1, self.in_channels, n_frames, dtype=torch.float).to(c.device)
        x = self._noise_path(noise.contiguous())
        total_length = c.size(2) * self.upsample_factor
        if x.size(2) > c.size(2):  # replicate-pad the conditioning up to the noise length (data movement)
            c = torch.cat([c, c[:, :, -1:].expand(-1, -1, x.size(2) - c.size(2))], dim=2).contiguous()
        y = self._body(x, c)[..., :total_length]
        return y.squeeze(0).transpose(1, 0)


class DiscreteSymbolStyleMelGANGenerator(torch.nn.Module):
    """models/style_melgan.py:364-602: StyleMelGAN over discrete units (HuBERT codes).  The symbol embedding plus the
    speaker embedding of each item's first frame is the conditioning, written channel-major by one embed launch
    (pwgb_symbol_embed_forward) that reads the index tensor in place; the noise path and the body are
    StyleMelGANGenerator's.  ``inference`` crops the upsampled noise to the T frames of the units instead of padding the
    conditioning, so the first block's InstanceNorm sees exactly T frames, as in the reference.  There is no
    ``register_stats``, as in the reference."""

    def __init__(
        self,
        in_channels=128,
        aux_channels=128,
        channels=64,
        out_channels=1,
        num_embs=100,
        num_spk_embs=128,
        spk_emb_dim=128,
        concat_spk_emb=False,
        kernel_size=9,
        dilation=2,
        bias=True,
        noise_upsample_scales=[11, 2, 2, 2],
        noise_upsample_activation="LeakyReLU",
        noise_upsample_activation_params={"negative_slope": 0.2},
        upsample_scales=[2, 2, 2, 2, 2, 2, 2, 2, 1],
        upsample_mode="nearest",
        gated_function="softmax",
        use_weight_norm=True,
    ):
        super().__init__()
        self.in_channels = in_channels
        self.num_spk_embs = num_spk_embs
        self.emb = torch.nn.Embedding(num_embeddings=num_embs, embedding_dim=aux_channels)
        self.spk_emb = torch.nn.Embedding(num_embeddings=num_spk_embs, embedding_dim=spk_emb_dim)
        self.concat_spk_emb = concat_spk_emb
        if not concat_spk_emb:
            assert aux_channels == spk_emb_dim
        else:
            aux_channels = aux_channels + spk_emb_dim
        self._build(aux_channels, channels, out_channels, kernel_size, dilation, bias, noise_upsample_scales, noise_upsample_activation,
                    noise_upsample_activation_params, upsample_scales, upsample_mode, gated_function)
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    remove_weight_norm = _GeneratorBase.remove_weight_norm
    _build = StyleMelGANGenerator._build
    apply_weight_norm = StyleMelGANGenerator.apply_weight_norm
    reset_parameters = StyleMelGANGenerator.reset_parameters
    _noise_path = StyleMelGANGenerator._noise_path
    _body = StyleMelGANGenerator._body
    _prep_symbols = DiscreteSymbolHiFiGANGenerator._prep_symbols

    def _check_input(self, c):
        assert c.size(1) == 2
        if self.concat_spk_emb:
            # style_melgan.py:493-495 concatenates the speaker embedding along time, so the first TADE aux conv, built
            # for aux_channels + spk_emb_dim, receives aux_channels: the reference fails there; so does the mirror
            raise PwgbError(f"concat_spk_emb=True: the first TADE aux conv expects {self.blocks[0].tade1.aux_conv[0].in_channels} "
                            f"channels, the embedding has {self.emb.embedding_dim} (the reference concatenates the speaker "
                            f"embedding along time)")

    def _embed(self, c):
        """(B, 2, T) symbol and speaker indices of any dtype -> (B, aux_channels, T) conditioning (see ops.symbol_embed)."""
        return ops.symbol_embed(c, self.emb.weight, self.spk_emb.weight)

    def forward(self, c, z=None):
        """c (B, 2, T) (symbol, speaker id) [, z (B, in_channels, T_z)] -> (B, out_channels, T * prod(upsample_scales))
        (style_melgan.py:474-508).  The noise path makes T_z * noise_upsample_factor frames and nothing crops it, so T
        must equal that (the default z has T_z = 1)."""
        self._check_input(c)
        if z is None:
            z = torch.randn(c.size(0), self.in_channels, 1).to(device=c.device, dtype=torch.float32)
        if c.size(2) != z.size(2) * self.noise_upsample_factor:
            raise PwgbError(f"{c.size(2)} frames of units, but the noise path makes {z.size(2) * self.noise_upsample_factor} "
                            f"({z.size(2)} noise frames x {self.noise_upsample_factor}); forward neither crops nor pads")
        return self._body(self._noise_path(z), self._embed(c))

    def inference(self, c, g=None, normalize_before=False, noise=None):
        """(T, 2) indices, or (T, 1) with a speaker id ``g`` -> (T * prod(upsample_scales), out_channels)
        (style_melgan.py:563-602).  ``noise`` (1, in_channels, (T - 1) // noise_upsample_factor + 1) may be passed for
        reproducibility; the upsampled noise is cropped to T frames."""
        assert not normalize_before, "No statistics are used."
        c = self._prep_symbols(c, g)
        self._check_input(c)
        T = c.size(2)
        n_frames = (T - 1) // self.noise_upsample_factor + 1
        if noise is None:
            noise = torch.randn(1, self.in_channels, n_frames, dtype=torch.float).to(c.device)
        elif tuple(noise.shape) != (1, self.in_channels, n_frames):
            raise PwgbError(f"inference: noise must be {(1, self.in_channels, n_frames)} for {T} frames, got {tuple(noise.shape)}")
        e = self._embed(c)
        x = self._noise_path(noise.contiguous())
        if x.size(2) > T:  # crop the noise path to the units (data movement)
            x = x[:, :, :T].contiguous()
        return self._body(x, e).squeeze(0).transpose(1, 0)


class ParallelWaveGANGenerator(_GeneratorBase):
    """models/parallel_wavegan.py:21-261."""

    def __init__(
        self,
        in_channels=1,
        out_channels=1,
        kernel_size=3,
        layers=30,
        stacks=3,
        residual_channels=64,
        gate_channels=128,
        skip_channels=64,
        aux_channels=80,
        aux_context_window=2,
        dropout=0.0,
        bias=True,
        use_weight_norm=True,
        use_causal_conv=False,
        upsample_conditional_features=True,
        upsample_net="ConvInUpsampleNetwork",
        upsample_params={"upsample_scales": [4, 4, 4, 4]},
    ):
        super().__init__()
        import math

        from . import layers as L

        self.in_channels = in_channels
        self.out_channels = out_channels
        self.aux_channels = aux_channels
        self.aux_context_window = aux_context_window
        self.layers = layers
        self.stacks = stacks
        self.kernel_size = kernel_size
        self.dropout = dropout
        self.use_causal_conv = use_causal_conv
        assert layers % stacks == 0
        layers_per_stack = layers // stacks
        self.first_conv = L.Conv1d1x1(in_channels, residual_channels, bias=True)
        upsample_params = dict(upsample_params)
        if upsample_conditional_features:
            upsample_params.update({"use_causal_conv": use_causal_conv})
            if upsample_net == "MelGANGenerator":
                assert aux_context_window == 0
                upsample_params.update({"use_weight_norm": False, "use_final_nonlinear_activation": False})
                self.upsample_net = MelGANGenerator(**upsample_params)
            else:
                if upsample_net == "ConvInUpsampleNetwork":
                    upsample_params.update({"aux_channels": aux_channels, "aux_context_window": aux_context_window})
                self.upsample_net = getattr(L, upsample_net)(**upsample_params)
            self.upsample_factor = int(np.prod(upsample_params["upsample_scales"]))
        else:
            self.upsample_net = None
            self.upsample_factor = 1
        self.conv_layers = torch.nn.ModuleList()
        for layer in range(layers):
            dilation = 2 ** (layer % layers_per_stack)
            self.conv_layers += [
                L.WaveNetResidualBlock(
                    kernel_size=kernel_size, residual_channels=residual_channels, gate_channels=gate_channels,
                    skip_channels=skip_channels, aux_channels=aux_channels, dilation=dilation, dropout=dropout,
                    bias=bias, use_causal_conv=use_causal_conv,
                )
            ]
        self.last_conv_layers = torch.nn.ModuleList(
            [
                torch.nn.ReLU(inplace=True),
                L.Conv1d1x1(skip_channels, skip_channels, bias=True),
                torch.nn.ReLU(inplace=True),
                L.Conv1d1x1(skip_channels, out_channels, bias=True),
            ]
        )
        self._skip_scale = math.sqrt(1.0 / layers)
        self._aux_pad = (aux_channels + 31) // 32 * 32
        if use_weight_norm:
            self.apply_weight_norm()

    def forward(self, z, c):
        """z: (B, 1, T) noise, c: (B, aux, T') -> (B, out_channels, T)  (parallel_wavegan.py:144-173)."""
        if c is not None and self.upsample_net is not None:
            if isinstance(self.upsample_net, MelGANGenerator):
                c = self.upsample_net(c)
            else:
                c = self.upsample_net(c, out_channels=self._aux_pad)
            assert c.size(-1) == z.size(-1)
        if c is not None and c.shape[1] != self._aux_pad:
            cp = torch.zeros((c.shape[0], self._aux_pad, c.shape[2]), device=c.device, dtype=c.dtype)
            cp[:, : c.shape[1]].copy_(c)
            c = cp
        fc = self.first_conv
        train = torch.is_grad_enabled() and next(self.parameters()).requires_grad
        skips = None if train else self._forward_packed(z, c)
        if skips is None:
            x = ops.conv1d(z, effective_weight(fc), fc.bias)
        if train:
            from .autograd import ScaledSumFn  # training: differentiable layer composition

            hs = []
            for f in self.conv_layers:
                x, h = f._forward_train(x, c)
                hs.append(h)
            skips = ScaledSumFn.apply(self._skip_scale, *hs)
            l1, l3 = self.last_conv_layers[1], self.last_conv_layers[3]
            h = ops.conv1d(skips, effective_weight(l1), l1.bias, pre_slope=0.0)
            return ops.conv1d(h, effective_weight(l3), l3.bias, pre_slope=0.0)
        if skips is None:
            skips = torch.zeros((x.shape[0], self.conv_layers[0].conv1x1_skip.out_channels, x.shape[2]), device=x.device, dtype=torch.float32)
            for f in self.conv_layers:
                x, _ = f(x, c, skips)
        # relu(a * s) = a * relu(s) for a > 0: the sqrt(1/layers) scale is folded into the 1x1 weights
        l1, l3 = self.last_conv_layers[1], self.last_conv_layers[3]
        h = ops.conv1d(skips, effective_weight(l1) * self._skip_scale, l1.bias, pre_slope=0.0)
        return ops.conv1d(h, effective_weight(l3), l3.bias, pre_slope=0.0)

    def _forward_packed(self, z, c):
        """Inference fast path: the residual stack as fused one-kernel layers on the packed (bf16 hi/lo operand
        layout) residual stream -- pwgb_wnstack_*.  Returns the skip sum (B, S, T) or None when the configuration
        has no fused kernel or dropout applies (train mode, also under no_grad): the caller then runs the per-layer
        fp32 path."""
        if c is None or (self.training and self.dropout > 0):
            return None
        l0 = self.conv_layers[0]
        G, R, K = l0.conv.out_channels, l0.conv.in_channels, l0.conv.kernel_size[0]
        S = l0.conv1x1_skip.out_channels
        A = self.aux_channels
        B, _, T = z.shape
        dmax = max(f.dilation for f in self.conv_layers)
        causal = self.use_causal_conv
        if c.shape[1] < A or not ops.WnStack.supported(B, T, R, G, S, A, K, dmax, causal):
            return None
        cache = self.__dict__.setdefault("_wn_stacks", {})
        key = (B, T, str(z.device))
        st = cache.get(key)
        if st is None:
            if len(cache) >= 4:
                cache.clear()
            st = cache[key] = ops.WnStack(B, T, R, G, S, A, K, dmax, z.device, causal)
        st.cur = 0
        st.pack_c(c)
        fc = self.first_conv
        st.first_conv(z, effective_weight(fc), fc.bias)
        skips = torch.empty((B, S, T), device=z.device, dtype=torch.float32)
        n = len(self.conv_layers)
        for i, f in enumerate(self.conv_layers):
            k = ops.param_key(f.conv, f.conv1x1_aux, f.conv1x1_skip, f.conv1x1_out)
            ent = f._cache.get("wnp")
            if ent is None or ent[0] != k:
                packed, bso = ops.wavenet_packed_weights(effective_weight(f.conv), effective_weight(f.conv1x1_aux), effective_weight(f.conv1x1_skip),
                                                         effective_weight(f.conv1x1_out), f.conv1x1_skip.bias, f.conv1x1_out.bias, A,
                                                         cache=f._cache, key=k, causal=causal)
            else:
                packed, bso = ent[1], ent[2]
            st.layer(packed, f.conv.bias, bso, f.dilation, skips, skips_init=(i == 0), write_x=(i < n - 1))
        return skips

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.Conv2d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    @staticmethod
    def _get_receptive_field_size(layers, stacks, kernel_size, dilation=lambda x: 2**x):
        assert layers % stacks == 0
        layers_per_cycle = layers // stacks
        dilations = [dilation(i % layers_per_cycle) for i in range(layers)]
        return (kernel_size - 1) * sum(dilations) + 1

    @property
    def receptive_field_size(self):
        return self._get_receptive_field_size(self.layers, self.stacks, self.kernel_size)

    def inference(self, c=None, x=None, normalize_before=False):
        """c: (T', aux) | None, x: (T, 1) noise | None -> (T, out_channels)  (parallel_wavegan.py:229-261)."""
        dev = next(self.parameters()).device
        if x is not None:
            if not isinstance(x, torch.Tensor):
                x = torch.tensor(x, dtype=torch.float).to(dev)
            x = x.transpose(1, 0).unsqueeze(0).contiguous()
        else:
            assert c is not None
            x = torch.randn(1, 1, len(c) * self.upsample_factor).to(dev)
        if c is not None:
            if not isinstance(c, torch.Tensor):
                c = torch.tensor(c, dtype=torch.float).to(dev)
            if normalize_before:
                c = (c - self.mean) / self.scale
            c = c.transpose(1, 0).unsqueeze(0)
            # ReplicationPad1d(aux_context_window): pure index gather of the edge frames
            w = self.aux_context_window
            idx = torch.arange(-w, c.shape[-1] + w, device=c.device).clamp_(0, c.shape[-1] - 1)
            c = c[:, :, idx].contiguous()
        return self.forward(x, c).squeeze(0).transpose(1, 0)


# ==========================================================================
# Discriminators (forward: every layer is one fused conv launch -- bias, LeakyReLU and the
# padding policy live inside the kernel; feature maps are written exactly once)
# ==========================================================================
import copy  # noqa: E402


class _NormMixin:
    def remove_weight_norm(self):
        def _remove_weight_norm(m):
            try:
                torch.nn.utils.remove_weight_norm(m)
            except ValueError:
                return

        self.apply(_remove_weight_norm)

    def remove_spectral_norm(self):
        def _remove_spectral_norm(m):
            try:
                torch.nn.utils.remove_spectral_norm(m)
            except ValueError:
                return

        self.apply(_remove_spectral_norm)


class ParallelWaveGANDiscriminator(torch.nn.Module, _NormMixin):
    """models/parallel_wavegan.py:264-371."""

    def __init__(self, in_channels=1, out_channels=1, kernel_size=3, layers=10, conv_channels=64, dilation_factor=1,
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.2}, bias=True,
                 use_weight_norm=True):
        super().__init__()
        from . import layers as L

        assert (kernel_size - 1) % 2 == 0, "Not support even number kernel size."
        assert dilation_factor > 0, "Dilation factor must be > 0."
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        self.conv_layers = torch.nn.ModuleList()
        conv_in_channels = in_channels
        for i in range(layers - 1):
            if i == 0:
                dilation = 1
            else:
                dilation = i if dilation_factor == 1 else dilation_factor**i
                conv_in_channels = conv_channels
            padding = (kernel_size - 1) // 2 * dilation
            self.conv_layers += [
                L.Conv1d(conv_in_channels, conv_channels, kernel_size=kernel_size, padding=padding, dilation=dilation, bias=bias),
                getattr(torch.nn, nonlinear_activation)(inplace=True, **nonlinear_activation_params),
            ]
        self.conv_layers += [L.Conv1d(conv_in_channels, out_channels, kernel_size=kernel_size, padding=(kernel_size - 1) // 2, bias=bias)]
        if use_weight_norm:
            self.apply_weight_norm()

    def forward(self, x):
        """(B, 1, T) -> (B, 1, T)."""
        mods = list(self.conv_layers)
        for i, m in enumerate(mods):
            if isinstance(m, torch.nn.Conv1d):
                act = i + 1 < len(mods) and not isinstance(mods[i + 1], torch.nn.Conv1d)
                x = ops.conv1d(x, effective_weight(m), m.bias, padding=m.padding[0], dilation=m.dilation[0],
                               post_act="lrelu" if act else None, post_slope=self.slope)
        return x

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.Conv2d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)


class ResidualParallelWaveGANDiscriminator(torch.nn.Module, _NormMixin):
    """models/parallel_wavegan.py:374-513: LReLU(1x1) -> WaveNet blocks without conditioning -> skip sum * sqrt(1/L)
    -> LReLU -> 1x1 -> LReLU -> 1x1.  The LeakyReLU after first_conv runs in its epilogue; sqrt(1/L) is folded into
    the first tail conv (LeakyReLU is positively homogeneous: lrelu(a s) = a lrelu(s) for a > 0)."""

    def __init__(self, in_channels=1, out_channels=1, kernel_size=3, layers=30, stacks=3, residual_channels=64,
                 gate_channels=128, skip_channels=64, dropout=0.0, bias=True, use_weight_norm=True, use_causal_conv=False,
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.2}):
        super().__init__()
        import math

        from . import layers as L

        assert (kernel_size - 1) % 2 == 0, "Not support even number kernel size."
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.layers = layers
        self.stacks = stacks
        self.kernel_size = kernel_size
        assert layers % stacks == 0
        layers_per_stack = layers // stacks
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        self.first_conv = torch.nn.Sequential(
            L.Conv1d1x1(in_channels, residual_channels, bias=True),
            getattr(torch.nn, nonlinear_activation)(inplace=True, **nonlinear_activation_params),
        )
        self.conv_layers = torch.nn.ModuleList()
        for layer in range(layers):
            self.conv_layers += [
                L.WaveNetResidualBlock(
                    kernel_size=kernel_size, residual_channels=residual_channels, gate_channels=gate_channels,
                    skip_channels=skip_channels, aux_channels=-1, dilation=2 ** (layer % layers_per_stack), dropout=dropout,
                    bias=bias, use_causal_conv=use_causal_conv,
                )
            ]
        self.last_conv_layers = torch.nn.ModuleList(
            [
                getattr(torch.nn, nonlinear_activation)(inplace=True, **nonlinear_activation_params),
                L.Conv1d1x1(skip_channels, skip_channels, bias=True),
                getattr(torch.nn, nonlinear_activation)(inplace=True, **nonlinear_activation_params),
                L.Conv1d1x1(skip_channels, out_channels, bias=True),
            ]
        )
        self._skip_scale = math.sqrt(1.0 / layers)
        if use_weight_norm:
            self.apply_weight_norm()

    def forward(self, x):
        """(B, in_channels, T) -> (B, out_channels, T)."""
        fc = self.first_conv[0]
        x = ops.conv1d(x, effective_weight(fc), fc.bias, post_act="lrelu", post_slope=self.slope)
        l1, l3 = self.last_conv_layers[1], self.last_conv_layers[3]
        if torch.is_grad_enabled() and (x.requires_grad or next(self.parameters()).requires_grad):
            from .autograd import ScaledSumFn

            hs = []
            for f in self.conv_layers:
                x, h = f._forward_train(x, None)
                hs.append(h)
            h = ops.conv1d(ScaledSumFn.apply(self._skip_scale, *hs), effective_weight(l1), l1.bias, pre_slope=self.slope)
        else:
            skips = torch.zeros((x.shape[0], self.conv_layers[0].conv1x1_skip.out_channels, x.shape[2]), device=x.device,
                                dtype=torch.float32)
            for f in self.conv_layers:
                x, _ = f(x, None, skips)
            h = ops.conv1d(skips, effective_weight(l1) * self._skip_scale, l1.bias, pre_slope=self.slope)
        return ops.conv1d(h, effective_weight(l3), l3.bias, pre_slope=self.slope)

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.Conv2d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)


class HiFiGANPeriodDiscriminator(torch.nn.Module, _NormMixin):
    """models/hifigan.py:270-401.  The (B, C, T/P, P) Conv2d (k,1) stack runs as period-strided 1-D
    convs directly on the flat waveform: the reflect extension to a multiple of P and the view are
    index arithmetic inside the kernel's tile loader (no padded copy)."""

    def __init__(self, in_channels=1, out_channels=1, period=3, kernel_sizes=[5, 3], channels=32,
                 downsample_scales=[3, 3, 3, 3, 1], max_downsample_channels=1024, bias=True,
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                 use_weight_norm=True, use_spectral_norm=False):
        super().__init__()
        assert len(kernel_sizes) == 2
        assert kernel_sizes[0] % 2 == 1, "Kernel size must be odd number."
        assert kernel_sizes[1] % 2 == 1, "Kernel size must be odd number."
        self.period = period
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        self.convs = torch.nn.ModuleList()
        in_chs, out_chs = in_channels, channels
        for downsample_scale in downsample_scales:
            self.convs += [
                torch.nn.Sequential(
                    torch.nn.Conv2d(in_chs, out_chs, (kernel_sizes[0], 1), (downsample_scale, 1), padding=((kernel_sizes[0] - 1) // 2, 0)),
                    getattr(torch.nn, nonlinear_activation)(**nonlinear_activation_params),
                )
            ]
            in_chs = out_chs
            out_chs = min(out_chs * 4, max_downsample_channels)
        self.output_conv = torch.nn.Conv2d(out_chs, out_channels, (kernel_sizes[1] - 1, 1), 1, padding=((kernel_sizes[1] - 1) // 2, 0))
        if use_weight_norm and use_spectral_norm:
            raise ValueError("Either use use_weight_norm or use_spectral_norm.")
        if use_weight_norm:
            self.apply_weight_norm()
        if use_spectral_norm:
            self.apply_spectral_norm()

    def forward(self, x):
        """(B, in_channels, T) -> list of per-layer outputs (4-D) + flattened logits."""
        outs = []
        for layer in self.convs:
            m = layer[0]
            x = ops.conv1d(x, effective_weight(m), m.bias, stride=m.stride[0], padding=m.padding[0], period=self.period,
                           post_act="lrelu", post_slope=self.slope)
            outs += [x]
        m = self.output_conv
        x = ops.conv1d(x, effective_weight(m), m.bias, stride=1, padding=m.padding[0], period=self.period)
        outs += [torch.flatten(x, 1, -1)]
        return outs

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, torch.nn.Conv2d):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def apply_spectral_norm(self):
        def _apply_spectral_norm(m):
            if isinstance(m, torch.nn.Conv2d):
                torch.nn.utils.spectral_norm(m)

        self.apply(_apply_spectral_norm)


class HiFiGANMultiPeriodDiscriminator(torch.nn.Module):
    """models/hifigan.py:404-453."""

    def __init__(self, periods=[2, 3, 5, 7, 11], discriminator_params={
        "in_channels": 1, "out_channels": 1, "kernel_sizes": [5, 3], "channels": 32,
        "downsample_scales": [3, 3, 3, 3, 1], "max_downsample_channels": 1024, "bias": True,
        "nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1},
        "use_weight_norm": True, "use_spectral_norm": False,
    }):
        super().__init__()
        self.discriminators = torch.nn.ModuleList()
        for period in periods:
            params = copy.deepcopy(discriminator_params)
            params["period"] = period
            self.discriminators += [HiFiGANPeriodDiscriminator(**params)]

    def forward(self, x):
        return [f(x) for f in self.discriminators]


class HiFiGANScaleDiscriminator(torch.nn.Module, _NormMixin):
    """models/hifigan.py:456-702 (including the load pre-hook that strips wn / sn when the
    checkpoint was trained without them, hifigan.py:647-702)."""

    def __init__(self, in_channels=1, out_channels=1, kernel_sizes=[15, 41, 5, 3], channels=128,
                 max_downsample_channels=1024, max_groups=16, bias=True, downsample_scales=[2, 2, 4, 4, 1],
                 nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1},
                 use_weight_norm=True, use_spectral_norm=False):
        super().__init__()
        self.layers = torch.nn.ModuleList()
        assert len(kernel_sizes) == 4
        for ks in kernel_sizes:
            assert ks % 2 == 1
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        act = getattr(torch.nn, nonlinear_activation)
        self.layers += [
            torch.nn.Sequential(
                torch.nn.Conv1d(in_channels, channels, kernel_sizes[0], bias=bias, padding=(kernel_sizes[0] - 1) // 2),
                act(**nonlinear_activation_params),
            )
        ]
        in_chs = channels
        out_chs = channels
        groups = 4
        for downsample_scale in downsample_scales:
            self.layers += [
                torch.nn.Sequential(
                    torch.nn.Conv1d(in_chs, out_chs, kernel_size=kernel_sizes[1], stride=downsample_scale,
                                    padding=(kernel_sizes[1] - 1) // 2, groups=groups, bias=bias),
                    act(**nonlinear_activation_params),
                )
            ]
            in_chs = out_chs
            out_chs = min(in_chs * 2, max_downsample_channels)
            groups = min(groups * 4, max_groups)
        out_chs = min(in_chs * 2, max_downsample_channels)
        self.layers += [
            torch.nn.Sequential(
                torch.nn.Conv1d(in_chs, out_chs, kernel_size=kernel_sizes[2], stride=1, padding=(kernel_sizes[2] - 1) // 2, bias=bias),
                act(**nonlinear_activation_params),
            )
        ]
        self.layers += [torch.nn.Conv1d(out_chs, out_channels, kernel_size=kernel_sizes[3], stride=1, padding=(kernel_sizes[3] - 1) // 2, bias=bias)]
        if use_weight_norm and use_spectral_norm:
            raise ValueError("Either use use_weight_norm or use_spectral_norm.")
        self.use_weight_norm = use_weight_norm
        if use_weight_norm:
            self.apply_weight_norm()
        self.use_spectral_norm = use_spectral_norm
        if use_spectral_norm:
            self.apply_spectral_norm()
        self._register_load_state_dict_pre_hook(self._load_state_dict_pre_hook)

    def forward(self, x):
        """(B, 1, T) -> list of the outputs of every layer."""
        outs = []
        for f in self.layers:
            m, act = (f[0], True) if isinstance(f, torch.nn.Sequential) else (f, False)
            x = ops.conv1d(x, effective_weight(m), m.bias, stride=m.stride[0], padding=m.padding[0], groups=m.groups,
                           post_act="lrelu" if act else None, post_slope=self.slope)
            outs += [x]
        return outs

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, torch.nn.Conv1d):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def apply_spectral_norm(self):
        def _apply_spectral_norm(m):
            if isinstance(m, torch.nn.Conv1d):
                torch.nn.utils.spectral_norm(m)

        self.apply(_apply_spectral_norm)

    def _load_state_dict_pre_hook(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        current_module_keys = [x for x in state_dict.keys() if x.startswith(prefix)]
        if self.use_weight_norm and not any(["weight_g" in k for k in current_module_keys]):
            logging.warning("weight norm is not applied in the pretrained model but the current model uses it: removing it (hifigan.py:665-683)")
            self.remove_weight_norm()
            self.use_weight_norm = False
        if self.use_spectral_norm and not any(["weight_u" in k for k in current_module_keys]):
            logging.warning("spectral norm is not applied in the pretrained model but the current model uses it: removing it (hifigan.py:685-702)")
            self.remove_spectral_norm()
            self.use_spectral_norm = False


class HiFiGANMultiScaleDiscriminator(torch.nn.Module):
    """models/hifigan.py:705-777."""

    def __init__(self, scales=3, downsample_pooling="AvgPool1d",
                 downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
                 discriminator_params={
                     "in_channels": 1, "out_channels": 1, "kernel_sizes": [15, 41, 5, 3], "channels": 128,
                     "max_downsample_channels": 1024, "max_groups": 16, "bias": True,
                     "downsample_scales": [2, 2, 4, 4, 1], "nonlinear_activation": "LeakyReLU",
                     "nonlinear_activation_params": {"negative_slope": 0.1},
                 }, follow_official_norm=False):
        super().__init__()
        if downsample_pooling != "AvgPool1d":
            raise PwgbError(f"downsample_pooling={downsample_pooling!r} has no sm_90a kernel (AvgPool1d only)")
        self.discriminators = torch.nn.ModuleList()
        for i in range(scales):
            params = copy.deepcopy(discriminator_params)
            if follow_official_norm:
                params["use_weight_norm"] = i != 0
                params["use_spectral_norm"] = i == 0
            self.discriminators += [HiFiGANScaleDiscriminator(**params)]
        self.pooling = torch.nn.AvgPool1d(**downsample_pooling_params)  # parameter container

    def _pool(self, x):
        p = self.pooling
        k = p.kernel_size[0] if isinstance(p.kernel_size, tuple) else p.kernel_size
        s = p.stride[0] if isinstance(p.stride, tuple) else p.stride
        pad = p.padding[0] if isinstance(p.padding, tuple) else p.padding
        return ops.avg_pool1d(x, k, s, pad, p.count_include_pad)

    def forward(self, x):
        outs = []
        for i, f in enumerate(self.discriminators):
            outs += [f(x)]
            if i + 1 < len(self.discriminators):
                x = self._pool(x)
        return outs


class HiFiGANMultiScaleMultiPeriodDiscriminator(torch.nn.Module):
    """models/hifigan.py:780-864."""

    def __init__(self, scales=3, scale_downsample_pooling="AvgPool1d",
                 scale_downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 2},
                 scale_discriminator_params={
                     "in_channels": 1, "out_channels": 1, "kernel_sizes": [15, 41, 5, 3], "channels": 128,
                     "max_downsample_channels": 1024, "max_groups": 16, "bias": True,
                     "downsample_scales": [2, 2, 4, 4, 1], "nonlinear_activation": "LeakyReLU",
                     "nonlinear_activation_params": {"negative_slope": 0.1},
                 }, follow_official_norm=True, periods=[2, 3, 5, 7, 11],
                 period_discriminator_params={
                     "in_channels": 1, "out_channels": 1, "kernel_sizes": [5, 3], "channels": 32,
                     "downsample_scales": [3, 3, 3, 3, 1], "max_downsample_channels": 1024, "bias": True,
                     "nonlinear_activation": "LeakyReLU", "nonlinear_activation_params": {"negative_slope": 0.1},
                     "use_weight_norm": True, "use_spectral_norm": False,
                 }):
        super().__init__()
        self.msd = HiFiGANMultiScaleDiscriminator(scales=scales, downsample_pooling=scale_downsample_pooling,
                                                  downsample_pooling_params=scale_downsample_pooling_params,
                                                  discriminator_params=scale_discriminator_params,
                                                  follow_official_norm=follow_official_norm)
        self.mpd = HiFiGANMultiPeriodDiscriminator(periods=periods, discriminator_params=period_discriminator_params)

    def forward(self, x):
        """Multi-scale outputs followed by multi-period outputs (hifigan.py:850-864)."""
        return self.msd(x) + self.mpd(x)


class MelGANDiscriminator(torch.nn.Module):
    """models/melgan.py:260-396."""

    def __init__(self, in_channels=1, out_channels=1, kernel_sizes=[5, 3], channels=16, max_downsample_channels=1024,
                 bias=True, downsample_scales=[4, 4, 4, 4], nonlinear_activation="LeakyReLU",
                 nonlinear_activation_params={"negative_slope": 0.2}, pad="ReflectionPad1d", pad_params={}):
        super().__init__()
        self.layers = torch.nn.ModuleList()
        assert len(kernel_sizes) == 2
        assert kernel_sizes[0] % 2 == 1
        assert kernel_sizes[1] % 2 == 1
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        self.pad_mode = pad_mode_of(pad, pad_params)
        act = getattr(torch.nn, nonlinear_activation)
        k0 = int(np.prod(kernel_sizes))
        self.layers += [
            torch.nn.Sequential(
                getattr(torch.nn, pad)((k0 - 1) // 2, **pad_params),
                torch.nn.Conv1d(in_channels, channels, k0, bias=bias),
                act(**nonlinear_activation_params),
            )
        ]
        in_chs = channels
        for downsample_scale in downsample_scales:
            out_chs = min(in_chs * downsample_scale, max_downsample_channels)
            self.layers += [
                torch.nn.Sequential(
                    torch.nn.Conv1d(in_chs, out_chs, kernel_size=downsample_scale * 10 + 1, stride=downsample_scale,
                                    padding=downsample_scale * 5, groups=in_chs // 4, bias=bias),
                    act(**nonlinear_activation_params),
                )
            ]
            in_chs = out_chs
        out_chs = min(in_chs * 2, max_downsample_channels)
        self.layers += [
            torch.nn.Sequential(
                torch.nn.Conv1d(in_chs, out_chs, kernel_sizes[0], padding=(kernel_sizes[0] - 1) // 2, bias=bias),
                act(**nonlinear_activation_params),
            )
        ]
        self.layers += [torch.nn.Conv1d(out_chs, out_channels, kernel_sizes[1], padding=(kernel_sizes[1] - 1) // 2, bias=bias)]
        self.reset_parameters()

    def forward(self, x, lengths=None):
        """x (B, in_channels, T) -> the output of every layer.  ``lengths`` (a ragged batch): per-layer (B,) int32 device
        tensors of each item's valid rows at that layer's output, ``layer_lengths(samples)``; every layer then keeps
        each item +0.0 past its own end and pads it at its own end (pwgb_conv1d_ragged_forward)."""
        outs = []
        if lengths is not None and len(lengths) != len(self.layers):
            raise PwgbError(f"MelGANDiscriminator: {len(lengths)} layer lengths for {len(self.layers)} layers")
        for i, f in enumerate(self.layers):
            kw = {} if lengths is None else {"mask": _length_mask(lengths[i], x.shape[0], 1)}
            if isinstance(f, torch.nn.Sequential):
                m = [q for q in f if isinstance(q, torch.nn.Conv1d)][0]
                first = i == 0
                x = ops.conv1d(x, effective_weight(m), m.bias, stride=m.stride[0],
                               padding=(m.kernel_size[0] - 1) // 2 if first else m.padding[0],
                               pad_mode=self.pad_mode if first else "zero", groups=m.groups,
                               post_act="lrelu", post_slope=self.slope, **kw)
            else:
                x = ops.conv1d(x, effective_weight(f), f.bias, padding=f.padding[0], **kw)
            outs += [x]
        return outs

    def layer_lengths(self, lengths):
        """Each item's valid rows after every layer, from its sample counts ``lengths`` (an int tensor on any device):
        ceil(L / s) after a conv of stride s (output rows (L + 2 * 5s - (10s + 1)) // s + 1), unchanged otherwise."""
        out, L = [], lengths
        for f in self.layers:
            m = [q for q in f if isinstance(q, torch.nn.Conv1d)][0] if isinstance(f, torch.nn.Sequential) else f
            s = m.stride[0]
            L = torch.div(L + (s - 1), s, rounding_mode="floor") if s > 1 else L
            out.append(L)
        return out

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.02)

        self.apply(_reset_parameters)


class MelGANMultiScaleDiscriminator(torch.nn.Module, _NormMixin):
    """models/melgan.py:399-534."""

    def __init__(self, in_channels=1, out_channels=1, scales=3, downsample_pooling="AvgPool1d",
                 downsample_pooling_params={"kernel_size": 4, "stride": 2, "padding": 1, "count_include_pad": False},
                 kernel_sizes=[5, 3], channels=16, max_downsample_channels=1024, bias=True,
                 downsample_scales=[4, 4, 4, 4], nonlinear_activation="LeakyReLU",
                 nonlinear_activation_params={"negative_slope": 0.2}, pad="ReflectionPad1d", pad_params={},
                 use_weight_norm=True):
        super().__init__()
        if downsample_pooling != "AvgPool1d":
            raise PwgbError(f"downsample_pooling={downsample_pooling!r} has no sm_90a kernel (AvgPool1d only)")
        self.discriminators = torch.nn.ModuleList()
        for _ in range(scales):
            self.discriminators += [
                MelGANDiscriminator(in_channels=in_channels, out_channels=out_channels, kernel_sizes=kernel_sizes,
                                    channels=channels, max_downsample_channels=max_downsample_channels, bias=bias,
                                    downsample_scales=downsample_scales, nonlinear_activation=nonlinear_activation,
                                    nonlinear_activation_params=nonlinear_activation_params, pad=pad, pad_params=pad_params)
            ]
        self.pooling = torch.nn.AvgPool1d(**downsample_pooling_params)
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    _pool = HiFiGANMultiScaleDiscriminator._pool

    def forward(self, x):
        outs = []
        for i, f in enumerate(self.discriminators):
            outs += [f(x)]
            if i + 1 < len(self.discriminators):
                x = self._pool(x)
        return outs

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.02)

        self.apply(_reset_parameters)


class StyleMelGANDiscriminator(torch.nn.Module, _NormMixin):
    """models/style_melgan.py:243-378: random-window discriminators -- for every window size a random crop of the
    waveform (``np.random.randint(T - ws)``, the reference's host RNG call, style_melgan.py:330) goes through a PQMF
    analysis bank (1, 2, 4, 8 sub-bands) into a MelGANDiscriminator; repeated ``repeats`` times.  The crop is a view,
    the analysis one strided FIR launch, every discriminator layer one fused conv launch."""

    def __init__(
        self,
        repeats=2,
        window_sizes=[512, 1024, 2048, 4096],
        pqmf_params=[[1, None, None, None], [2, 62, 0.26700, 9.0], [4, 62, 0.14200, 9.0], [8, 62, 0.07949, 9.0]],
        discriminator_params={
            "out_channels": 1, "kernel_sizes": [5, 3], "channels": 16, "max_downsample_channels": 512, "bias": True,
            "downsample_scales": [4, 4, 4, 1], "nonlinear_activation": "LeakyReLU",
            "nonlinear_activation_params": {"negative_slope": 0.2}, "pad": "ReflectionPad1d", "pad_params": {},
        },
        use_weight_norm=True,
    ):
        super().__init__()
        from .layers import PQMF

        assert len(window_sizes) == len(pqmf_params)
        sizes = [ws // p[0] for ws, p in zip(window_sizes, pqmf_params)]
        assert len(window_sizes) == sum([sizes[0] == size for size in sizes])
        self.repeats = repeats
        self.window_sizes = window_sizes
        self.pqmfs = torch.nn.ModuleList()
        self.discriminators = torch.nn.ModuleList()
        for pqmf_param in pqmf_params:
            d_params = copy.deepcopy(discriminator_params)
            d_params["in_channels"] = pqmf_param[0]
            self.pqmfs += [torch.nn.Identity() if pqmf_param[0] == 1 else PQMF(*pqmf_param)]
            self.discriminators += [MelGANDiscriminator(**d_params)]
        if use_weight_norm:
            self.apply_weight_norm()
        self.reset_parameters()

    def forward(self, x):
        """(B, 1, T) -> list of repeats * #discriminators lists of feature maps (last = logits)."""
        outs = []
        for _ in range(self.repeats):
            outs += self._forward(x)
        return outs

    def _forward(self, x):
        outs = []
        for idx, (ws, pqmf, disc) in enumerate(zip(self.window_sizes, self.pqmfs, self.discriminators)):
            start_idx = np.random.randint(x.size(-1) - ws)
            x_ = x[:, :, start_idx : start_idx + ws].contiguous()
            x_ = pqmf(x_) if idx == 0 else pqmf.analysis(x_)
            outs += [disc(x_)]
        return outs

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    def reset_parameters(self):
        def _reset_parameters(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                m.weight.data.normal_(0.0, 0.02)

        self.apply(_reset_parameters)


class VQVAE(torch.nn.Module):
    """models/vqvae.py:16-185: wav2wav VQ-VAE.  The encoder (a MelGANDiscriminator in every recipe) gives z_e, its last
    output; one pwgb_vq_forward launch finds the nearest codes and writes both the quantised z_q and the decoder input
    -- the codes, the (embedded) local conditioning and the global embedding broadcast over time -- so neither
    ``torch.cat`` of the reference is built; the decoder is a MelGANGenerator.  State-dict keys follow the reference,
    including its quirks: ``local_embed`` is weight-normed like every Conv1d, ``global_embed`` is not, and with
    ``use_weight_norm=False`` the decoder keeps the weight norm MelGANGenerator applies by default."""

    def __init__(
        self,
        in_channels=1,
        out_channels=1,
        num_embeds=512,
        embed_dim=256,
        num_local_embeds=None,
        local_embed_dim=None,
        num_global_embeds=None,
        global_embed_dim=None,
        encoder_type="MelGANDiscriminator",
        decoder_type="MelGANGenerator",
        encoder_conf={"out_channels": 256, "downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 1024},
        decoder_conf={"in_channels": 256, "upsample_scales": [4, 4, 2, 2], "channels": 512, "stacks": 3},
        use_weight_norm=True,
    ):
        super().__init__()
        import sys

        mod = sys.modules[__name__]
        if not hasattr(mod, encoder_type) or not hasattr(mod, decoder_type):
            raise PwgbError(f"VQVAE: encoder_type={encoder_type!r} / decoder_type={decoder_type!r} are not mirrored")
        encoder_class = getattr(mod, encoder_type)
        decoder_class = getattr(mod, decoder_type)
        encoder_conf = dict(encoder_conf, in_channels=in_channels)
        decoder_conf = dict(decoder_conf, out_channels=out_channels)
        if not issubclass(decoder_class, MelGANGenerator):
            raise NotImplementedError(f"{decoder_class} is not supported yet.")
        self.in_channels = in_channels
        if num_local_embeds is not None:
            self.local_embed = torch.nn.Conv1d(num_local_embeds, local_embed_dim, 1) if local_embed_dim is not None else None
        if num_global_embeds is not None:
            self.global_embed = torch.nn.Embedding(num_global_embeds, global_embed_dim)
        self.encoder = encoder_class(**encoder_conf)
        self.codebook = VQCodebook(num_embeds=num_embeds, embed_dim=embed_dim)
        self.decoder = decoder_class(**decoder_conf)
        if use_weight_norm:
            self.remove_weight_norm()  # the decoder's own weight norm, as in the reference
            self.apply_weight_norm()

    def _local(self, l):
        if self.local_embed is None:
            return l
        m = self.local_embed
        return ops.conv1d(l, effective_weight(m), m.bias)

    def _global(self, g):
        return (self.global_embed.weight, g) if g is not None else (None, None)

    def _encode(self, x):
        z_e = self.encoder(x)
        return z_e[-1] if isinstance(z_e, list) else z_e

    def forward(self, x, l=None, g=None):
        """x (B, in_channels, T), l (B, num_local_embeds, T') or None, g (B,) int64 or None ->
        (x_bar (B, out_channels, T), z_e, z_q (B, embed_dim, T'))  (vqvae.py:80-110)."""
        z_e = self._encode(x)
        if l is not None:
            l = self._local(l)
        gt, g = self._global(g)
        dec, z_q, _ = ops.vq(z_e, self.codebook.embedding.weight, l=l, global_table=gt, g=g)
        return self.decoder(dec), z_e, z_q

    def encode(self, x, lengths=None):
        """x (B, in_channels, T) -> codebook indices (B, T')  (vqvae.py:112-125).

        ``lengths`` ((B,) int32 sample counts on the device): a ragged batch, x padded past each item's end.  Item b's
        first ceil(lengths[b] / hop) indices equal ``encode`` of that item alone (DESIGN.md §3.16); the later ones are
        the codes of zero frames, to be cropped."""
        if lengths is None:
            return self.codebook(self._encode(x))
        self._check_ragged(lengths, x.shape[-1], self.min_ragged_samples(), "encode")
        return self.codebook(self.encoder(x, self.encoder.layer_lengths(lengths))[-1])

    def decode(self, indices, l=None, g=None, lengths=None):
        """indices (B, T') int64 -> (B, out_channels, T)  (vqvae.py:127-147): gather and assembly only.

        ``lengths`` ((B,) int32 frame counts on the device): a ragged batch.  Indices past an item's end must still be
        codes (0 will do); samples before lengths[b] * hop equal ``decode`` of that item alone, the later ones are +0.0."""
        if lengths is not None:
            self._check_ragged(lengths, indices.shape[-1], self.min_ragged_frames(), "decode")
        return self._decode(indices, l, g, lengths)

    def _decode(self, indices, l, g, lengths):
        if l is not None:
            l = self._local(l)
        gt, g = self._global(g)
        _, _, dec = ops.vq_raw(None, self.codebook.embedding.weight, indices=indices, z_q=False, dec=True, l=l, global_table=gt, g=g)
        return self.decoder(dec) if lengths is None else self.decoder(dec, lengths)

    @property
    def hop(self):
        """Samples per code frame: the encoder's total stride."""
        return int(np.prod([f[0].stride[0] for f in self.encoder.layers[1:-2]]))

    def min_ragged_frames(self):
        """The fewest code frames a ragged decode takes: every reflect-padded conv of the decoder needs its pad < the
        item's length at its rate (ReflectionPad1d)."""
        dec = self.decoder
        need, rate = [(dec.kernel_size - 1) // 2 + 1], 1  # the input conv
        for m in dec.melgan:
            if isinstance(m, torch.nn.ConvTranspose1d):
                rate *= m.stride[0]
            elif isinstance(m, ResidualStack):
                need.append(-(-((m.kernel_size - 1) // 2 * m.dilation + 1) // rate))
        need.append(-(-((dec.kernel_size - 1) // 2 + 1) // rate))  # the output conv
        return max(need)

    def min_ragged_samples(self):
        """The shortest utterance a ragged batch converts: the encoder's reflect-padded input conv needs its pad < the
        length, and the decoder ``min_ragged_frames`` frames of ceil(length / hop)."""
        c0 = [q for q in self.encoder.layers[0] if isinstance(q, torch.nn.Conv1d)][0]
        return max((c0.kernel_size[0] - 1) // 2 + 1, (self.min_ragged_frames() - 1) * self.hop + 1)

    def _check_ragged(self, lengths, T, least, what):
        """the argument checks of a ragged encode / decode; the lengths are read on the host outside graph capture"""
        if not isinstance(self.encoder, MelGANDiscriminator) or not isinstance(self.decoder, MelGANGenerator):
            raise PwgbError("VQVAE: per-item lengths serve the MelGANDiscriminator encoder and MelGANGenerator decoder")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise PwgbError(f"VQVAE.{what}: per-item lengths are an inference feature (run under torch.no_grad)")
        if torch.cuda.is_current_stream_capturing():
            return
        host = [int(v) for v in lengths.tolist()]
        if any(L < least or L > T for L in host):
            raise PwgbError(f"VQVAE.{what}: lengths {host} must lie in [{least}, {T}] (the reflect pads need at least {least})")

    def apply_weight_norm(self):
        def _apply_weight_norm(m):
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                torch.nn.utils.weight_norm(m)

        self.apply(_apply_weight_norm)

    remove_weight_norm = _GeneratorBase.remove_weight_norm
