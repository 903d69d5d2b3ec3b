"""ctypes binding of include/pwgb.h (libpwgb.so).  Fails loudly if the library is absent."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libpwgb.so")

PAD_ZERO, PAD_REFLECT, PAD_REPLICATE = 0, 1, 2
ACT_NONE, ACT_TANH, ACT_LRELU = 0, 1, 2


class PwgbError(RuntimeError):
    pass


class Conv1dDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("cin", C.c_int32), ("cout", C.c_int32), ("t_in", C.c_int32), ("t_out", C.c_int32),
        ("kernel", C.c_int32), ("stride", C.c_int32), ("dilation", C.c_int32), ("groups", C.c_int32),
        ("pad_left", C.c_int32), ("pad_mode", C.c_int32), ("period", C.c_int32), ("t_valid", C.c_int32),
        ("pre_slope", C.c_float), ("pre_gate", C.c_int32), ("post_act", C.c_int32), ("post_slope", C.c_float),
        ("out_scale", C.c_float), ("accumulate", C.c_int32), ("shuffle", C.c_int32), ("shuffle_pad", C.c_int32),
        ("shuffle_tout", C.c_int32),
        ("x_batch_stride", C.c_int64), ("y_batch_stride", C.c_int64), ("r_batch_stride", C.c_int64),
    ]


class ConvTr1dDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("cin", C.c_int32), ("cout", C.c_int32), ("t_in", C.c_int32), ("t_out", C.c_int32),
        ("kernel", C.c_int32), ("stride", C.c_int32), ("padding", C.c_int32), ("pre_slope", C.c_float),
        ("groups", C.c_int32), ("period", C.c_int32),
    ]


class WaveNetDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("t", C.c_int32), ("residual_channels", C.c_int32), ("gate_channels", C.c_int32),
        ("skip_channels", C.c_int32), ("aux_channels", C.c_int32), ("kernel", C.c_int32), ("dilation", C.c_int32),
    ]


class ResBlockDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("channels", C.c_int32), ("t", C.c_int32), ("kernel", C.c_int32), ("dilation", C.c_int32),
        ("slope", C.c_float), ("out_scale", C.c_float), ("accumulate", C.c_int32),
    ]


class WnStackDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("t", C.c_int32), ("residual_channels", C.c_int32), ("gate_channels", C.c_int32),
        ("skip_channels", C.c_int32), ("aux_channels", C.c_int32), ("kernel", C.c_int32), ("halo", C.c_int32),
    ]


class StftDesc(C.Structure):
    _fields_ = [("batch", C.c_int32), ("t", C.c_int32), ("n_fft", C.c_int32), ("hop", C.c_int32),
                ("win_length", C.c_int32), ("clamp_eps", C.c_float)]


_lib = None


def lib():
    """Load libpwgb.so once.  No fallback: a missing library is a hard error."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PwgbError(
            f"{LIB_PATH} not found: the CUDA extension is not built. Run `python -c 'import __graft_entry__ as g; "
            "g.build()'` (needs nvcc). parallelwavegan_b200 has no CPU/PyTorch fallback."
        )
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.pwgb_last_error.restype = C.c_char_p
    L.pwgb_version.restype = C.c_int
    L.pwgb_compiled_arch.restype = C.c_int
    L.pwgb_launch_count.restype = C.c_longlong
    L.pwgb_reset_launch_count.restype = None
    L.pwgb_conv1d_forward.restype = C.c_int
    L.pwgb_conv1d_forward.argtypes = [C.POINTER(Conv1dDesc), vp, vp, vp, vp, vp, vp]
    L.pwgb_conv_transpose1d_workspace.restype = C.c_size_t
    L.pwgb_conv_transpose1d_workspace.argtypes = [C.POINTER(ConvTr1dDesc)]
    L.pwgb_conv_transpose1d_forward.restype = C.c_int
    L.pwgb_conv_transpose1d_forward.argtypes = [C.POINTER(ConvTr1dDesc), vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.pwgb_conv_transpose1d_cat_supported.restype = C.c_int
    L.pwgb_conv_transpose1d_cat_supported.argtypes = [C.POINTER(ConvTr1dDesc), C.c_int]
    L.pwgb_conv_transpose1d_cat_forward.restype = C.c_int
    L.pwgb_conv_transpose1d_cat_forward.argtypes = [C.POINTER(ConvTr1dDesc), C.c_int, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.pwgb_dropout_forward.restype = C.c_int
    L.pwgb_dropout_forward.argtypes = [vp, vp, C.c_longlong, C.c_float, C.c_ulonglong, C.c_ulonglong, vp]
    L.pwgb_dropout_backward.restype = C.c_int
    L.pwgb_dropout_backward.argtypes = [vp, vp, C.c_longlong, C.c_float, C.c_ulonglong, C.c_ulonglong, vp]
    L.pwgb_conv1d_tc_packed_weight_bytes.restype = C.c_size_t
    L.pwgb_conv1d_tc_packed_weight_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.pwgb_conv1d_tc_pack_weight.restype = C.c_int
    L.pwgb_conv1d_tc_pack_weight.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp]
    L.pwgb_conv1d_tc_pack_weight_grouped.restype = C.c_int
    L.pwgb_conv1d_tc_pack_weight_grouped.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    L.pwgb_conv1d_tc_supported.restype = C.c_int
    L.pwgb_conv1d_tc_supported.argtypes = [C.POINTER(Conv1dDesc)]
    L.pwgb_conv1d_tc_forward.restype = C.c_int
    L.pwgb_conv1d_tc_forward.argtypes = [C.POINTER(Conv1dDesc), vp, vp, vp, vp, vp, vp]
    L.pwgb_debug_set.restype = None
    L.pwgb_debug_set.argtypes = [C.c_int, C.c_int]
    L.pwgb_debug_get.restype = C.c_int
    L.pwgb_debug_get.argtypes = [C.c_int, vp, C.c_size_t]
    L.pwgb_resblock_pair_supported.restype = C.c_int
    L.pwgb_resblock_pair_supported.argtypes = [C.POINTER(ResBlockDesc)]
    L.pwgb_resblock_pair_plan.restype = C.c_int
    L.pwgb_resblock_pair_plan.argtypes = [C.POINTER(ResBlockDesc), C.POINTER(C.c_int)]
    L.pwgb_resblock_pair_variant.restype = C.c_int
    L.pwgb_resblock_pair_variant.argtypes = [C.POINTER(ResBlockDesc)]
    L.pwgb_resblock_pair_forward.restype = C.c_int
    L.pwgb_resblock_pair_forward.argtypes = [C.POINTER(ResBlockDesc), vp, vp, vp, vp, vp, vp, vp]
    L.pwgb_wavenet_supported.restype = C.c_int
    L.pwgb_wavenet_supported.argtypes = [C.POINTER(WaveNetDesc)]
    L.pwgb_wavenet_packed_bytes.restype = C.c_size_t
    L.pwgb_wavenet_packed_bytes.argtypes = [C.POINTER(WaveNetDesc)]
    L.pwgb_wavenet_pack.restype = C.c_int
    L.pwgb_wavenet_pack.argtypes = [C.POINTER(WaveNetDesc), vp, vp, C.c_int, vp, vp, vp, vp]
    L.pwgb_wavenet_layer_forward.restype = C.c_int
    L.pwgb_wavenet_layer_forward.argtypes = [C.POINTER(WaveNetDesc), vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.pwgb_wnstack_supported.restype = C.c_int
    L.pwgb_wnstack_supported.argtypes = [C.POINTER(WnStackDesc)]
    for fn in (L.pwgb_wnstack_x_bytes, L.pwgb_wnstack_c_bytes):
        fn.restype = C.c_size_t
        fn.argtypes = [C.POINTER(WnStackDesc)]
    L.pwgb_wnstack_pack_x.restype = C.c_int
    L.pwgb_wnstack_pack_x.argtypes = [C.POINTER(WnStackDesc), vp, vp, vp]
    L.pwgb_wnstack_unpack_x.restype = C.c_int
    L.pwgb_wnstack_unpack_x.argtypes = [C.POINTER(WnStackDesc), vp, vp, vp]
    L.pwgb_wnstack_pack_c.restype = C.c_int
    L.pwgb_wnstack_pack_c.argtypes = [C.POINTER(WnStackDesc), vp, C.c_longlong, vp, vp]
    L.pwgb_wnstack_first_conv.restype = C.c_int
    L.pwgb_wnstack_first_conv.argtypes = [C.POINTER(WnStackDesc), vp, C.c_int, vp, vp, vp, vp]
    L.pwgb_wnstack_layer_forward.restype = C.c_int
    L.pwgb_wnstack_layer_forward.argtypes = [C.POINTER(WnStackDesc), C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp]
    L.pwgb_collate_crop.restype = C.c_int
    L.pwgb_collate_crop.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.pwgb_prep_features.restype = C.c_int
    L.pwgb_prep_features.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.pwgb_pcm16_forward.restype = C.c_int
    L.pwgb_pcm16_forward.argtypes = [vp, vp, C.c_longlong, vp]
    L.pwgb_mt_clip_coef.restype = C.c_int
    L.pwgb_mt_clip_coef.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, vp, vp, vp]
    L.pwgb_mt_adam_step.restype = C.c_int
    L.pwgb_mt_adam_step.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int] + [C.c_float] * 7 + [vp, C.c_int, vp]
    for fn in (L.pwgb_s2d_forward, L.pwgb_s2d_backward):
        fn.restype = C.c_int
        fn.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_int, vp]
    L.pwgb_upsample_fir_forward.restype = C.c_int
    L.pwgb_upsample_fir_forward.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_longlong, vp]
    L.pwgb_mr_stft_loss_workspace.restype = C.c_size_t
    L.pwgb_mr_stft_loss_workspace.argtypes = [C.POINTER(StftDesc), C.c_int]
    L.pwgb_mr_stft_loss_forward.restype = C.c_int
    L.pwgb_mr_stft_loss_forward.argtypes = [C.POINTER(StftDesc), C.c_int, vp, vp, C.POINTER(vp), vp, vp, C.c_size_t, vp]
    L.pwgb_stft_amplitude_forward.restype = C.c_int
    L.pwgb_stft_amplitude_forward.argtypes = [C.POINTER(StftDesc), vp, vp, vp, vp, vp, vp]
    L.pwgb_mel_project_forward.restype = C.c_int
    L.pwgb_mel_project_forward.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_float, C.c_float, vp, vp, vp, vp]
    L.pwgb_reduce_mean_forward.restype = C.c_int
    L.pwgb_reduce_mean_forward.argtypes = [C.c_int, vp, vp, C.c_longlong, C.c_float, C.c_float, C.c_float, C.c_int, vp, vp, C.c_int, vp]
    L.pwgb_avg_pool1d_forward.restype = C.c_int
    L.pwgb_avg_pool1d_forward.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.pwgb_conv1d_wgrad_workspace.restype = C.c_size_t
    L.pwgb_conv1d_wgrad_workspace.argtypes = [C.POINTER(Conv1dDesc)]
    L.pwgb_conv1d_wgrad.restype = C.c_int
    L.pwgb_conv1d_wgrad.argtypes = [C.POINTER(Conv1dDesc), vp, vp, C.c_float, vp, C.c_int, vp, C.c_size_t, vp]
    L.pwgb_conv1d_wgrad_tc_supported.restype = C.c_int
    L.pwgb_conv1d_wgrad_tc_supported.argtypes = [C.POINTER(Conv1dDesc)]
    L.pwgb_conv1d_wgrad_tc_workspace.restype = C.c_size_t
    L.pwgb_conv1d_wgrad_tc_workspace.argtypes = [C.POINTER(Conv1dDesc)]
    L.pwgb_conv1d_wgrad_tc.restype = C.c_int
    L.pwgb_conv1d_wgrad_tc.argtypes = [C.POINTER(Conv1dDesc), vp, vp, C.c_float, vp, vp, C.c_size_t, vp]
    L.pwgb_act_backward.restype = C.c_int
    L.pwgb_act_backward.argtypes = [C.c_int, vp, vp, vp, C.c_longlong, C.c_float, C.c_float, C.c_int, vp]
    L.pwgb_bias_grad.restype = C.c_int
    L.pwgb_bias_grad.argtypes = [vp, vp, C.c_int, C.c_int, C.c_longlong, C.c_int, vp]
    L.pwgb_reduce_mean_backward.restype = C.c_int
    L.pwgb_reduce_mean_backward.argtypes = [C.c_int, vp, vp, C.c_longlong, C.c_float, C.c_float, C.c_float, vp, vp, C.c_int, vp]
    L.pwgb_avg_pool1d_backward.restype = C.c_int
    L.pwgb_avg_pool1d_backward.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.pwgb_axpby.restype = C.c_int
    L.pwgb_axpby.argtypes = [C.c_longlong, C.c_float, vp, C.c_float, vp, vp]
    L.pwgb_scaled_sum.restype = C.c_int
    L.pwgb_scaled_sum.argtypes = [vp, C.c_int, C.c_float, vp, C.c_longlong, C.c_int, vp]
    L.pwgb_instance_norm_forward.restype = C.c_int
    L.pwgb_instance_norm_forward.argtypes = [vp, vp, C.c_longlong, C.c_longlong, C.c_float, C.c_float, vp]
    L.pwgb_upsample_nearest_forward.restype = C.c_int
    L.pwgb_upsample_nearest_forward.argtypes = [vp, vp, C.c_longlong, C.c_longlong, C.c_int, vp]
    L.pwgb_leaky_relu_forward.restype = C.c_int
    L.pwgb_leaky_relu_forward.argtypes = [vp, vp, C.c_longlong, C.c_float, vp]
    L.pwgb_tade_combine_forward.restype = C.c_int
    L.pwgb_tade_combine_forward.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_longlong, C.c_int, vp]
    L.pwgb_tade_gate_forward.restype = C.c_int
    L.pwgb_tade_gate_forward.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, vp]
    for fn in (L.pwgb_pad1d_forward, L.pwgb_pad1d_backward):
        fn.restype = C.c_int
        fn.argtypes = [vp, vp, C.c_longlong, C.c_longlong, C.c_int, C.c_int, C.c_int, vp]
    L.pwgb_stft_amplitude_backward.restype = C.c_int
    L.pwgb_stft_amplitude_backward.argtypes = [C.POINTER(StftDesc), vp, vp, vp, vp, vp, vp]
    L.pwgb_mel_project_backward.restype = C.c_int
    L.pwgb_mel_project_backward.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_float, C.c_float, vp, vp, vp]
    L.pwgb_gate_forward.restype = C.c_int
    L.pwgb_gate_forward.argtypes = [vp, vp, C.c_int, C.c_int, C.c_longlong, vp]
    L.pwgb_gate_backward.restype = C.c_int
    L.pwgb_gate_backward.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_longlong, vp]
    L.pwgb_instance_norm_backward.restype = C.c_int
    L.pwgb_instance_norm_backward.argtypes = [vp, vp, vp, C.c_longlong, C.c_longlong, C.c_float, C.c_float, vp]
    L.pwgb_upsample_nearest_backward.restype = C.c_int
    L.pwgb_upsample_nearest_backward.argtypes = [vp, vp, C.c_longlong, C.c_longlong, C.c_int, vp]
    L.pwgb_tade_combine_backward.restype = C.c_int
    L.pwgb_tade_combine_backward.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_longlong, C.c_int, vp]
    L.pwgb_tade_gate_backward.restype = C.c_int
    L.pwgb_tade_gate_backward.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_longlong, C.c_int, vp]
    L.pwgb_upsample_fir_backward.restype = C.c_int
    L.pwgb_upsample_fir_backward.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_longlong, vp, vp, vp]
    L.pwgb_stft_loss_terms.restype = C.c_int
    L.pwgb_stft_loss_terms.argtypes = [vp, vp, C.c_longlong, C.c_float, C.c_int, vp, vp, vp, C.c_int, vp]
    L.pwgb_stft_loss_dmag.restype = C.c_int
    L.pwgb_stft_loss_dmag.argtypes = [vp, vp, C.c_longlong, vp, vp, C.c_float, vp, vp]
    ll = C.c_longlong
    L.pwgb_symbol_embed_forward.restype = C.c_int
    L.pwgb_symbol_embed_forward.argtypes = [vp, C.c_int, ll, ll, ll, vp, C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    L.pwgb_symbol_embed_backward_workspace.restype = C.c_size_t
    L.pwgb_symbol_embed_backward_workspace.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    L.pwgb_symbol_embed_backward.restype = C.c_int
    L.pwgb_symbol_embed_backward.argtypes = [vp, vp, vp, C.c_int, ll, ll, ll, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int,
                                             vp, vp, C.c_size_t, vp]
    L.pwgb_channel_layernorm_forward.restype = C.c_int
    L.pwgb_channel_layernorm_forward.argtypes = [vp, vp, vp, C.c_int, C.c_int, ll, C.c_float, vp, vp, vp, vp]
    L.pwgb_channel_layernorm_backward_workspace.restype = C.c_size_t
    L.pwgb_channel_layernorm_backward_workspace.argtypes = [C.c_int, C.c_int, ll]
    L.pwgb_channel_layernorm_backward.restype = C.c_int
    L.pwgb_channel_layernorm_backward.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int, ll, vp, vp, vp, vp, C.c_size_t, vp]
    L.pwgb_duration_loss_forward.restype = C.c_int
    L.pwgb_duration_loss_forward.argtypes = [vp, vp, ll, C.c_float, vp, vp]
    L.pwgb_duration_loss_backward.restype = C.c_int
    L.pwgb_duration_loss_backward.argtypes = [vp, vp, ll, C.c_float, vp, vp, vp]
    L.pwgb_duration_round.restype = C.c_int
    L.pwgb_duration_round.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_float, C.c_int, vp]
    L.pwgb_collate_runlength.restype = C.c_int
    L.pwgb_collate_runlength.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_int, ll, vp]
    L.pwgb_vq_forward.restype = C.c_int
    L.pwgb_vq_forward.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    L.pwgb_vq_backward.restype = C.c_int
    L.pwgb_vq_backward.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, vp, vp]
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        msg = lib().pwgb_last_error().decode("utf-8", "replace")
        raise PwgbError(f"{what} failed (status {rc}): {msg}")


def launch_count():
    return int(lib().pwgb_launch_count())


def reset_launch_count():
    lib().pwgb_reset_launch_count()


EXPORTED_SYMBOLS = [
    "pwgb_last_error", "pwgb_version", "pwgb_compiled_arch", "pwgb_launch_count", "pwgb_reset_launch_count",
    "pwgb_conv1d_forward", "pwgb_conv_transpose1d_workspace", "pwgb_conv_transpose1d_forward",
    "pwgb_conv_transpose1d_cat_supported", "pwgb_conv_transpose1d_cat_forward", "pwgb_dropout_forward", "pwgb_dropout_backward",
    "pwgb_conv1d_tc_packed_weight_bytes", "pwgb_conv1d_tc_pack_weight", "pwgb_conv1d_tc_pack_weight_grouped",
    "pwgb_conv1d_tc_supported",
    "pwgb_conv1d_tc_forward", "pwgb_debug_set", "pwgb_debug_get",
    "pwgb_resblock_pair_supported", "pwgb_resblock_pair_plan", "pwgb_resblock_pair_variant", "pwgb_resblock_pair_forward",
    "pwgb_wavenet_supported", "pwgb_wavenet_packed_bytes",
    "pwgb_wavenet_pack", "pwgb_wavenet_layer_forward", "pwgb_upsample_fir_forward",
    "pwgb_s2d_forward", "pwgb_s2d_backward", "pwgb_mt_clip_coef", "pwgb_mt_adam_step", "pwgb_prep_features", "pwgb_pcm16_forward", "pwgb_collate_crop",
    "pwgb_wnstack_supported", "pwgb_wnstack_x_bytes", "pwgb_wnstack_c_bytes", "pwgb_wnstack_pack_x", "pwgb_wnstack_unpack_x",
    "pwgb_wnstack_pack_c", "pwgb_wnstack_first_conv", "pwgb_wnstack_layer_forward",
    "pwgb_mr_stft_loss_workspace", "pwgb_mr_stft_loss_forward", "pwgb_stft_amplitude_forward",
    "pwgb_mel_project_forward", "pwgb_reduce_mean_forward", "pwgb_avg_pool1d_forward",
    "pwgb_conv1d_wgrad_workspace", "pwgb_conv1d_wgrad", "pwgb_conv1d_wgrad_tc_supported",
    "pwgb_conv1d_wgrad_tc_workspace", "pwgb_conv1d_wgrad_tc", "pwgb_act_backward", "pwgb_bias_grad",
    "pwgb_reduce_mean_backward", "pwgb_avg_pool1d_backward", "pwgb_axpby", "pwgb_scaled_sum", "pwgb_pad1d_forward", "pwgb_pad1d_backward",
    "pwgb_instance_norm_forward", "pwgb_upsample_nearest_forward", "pwgb_leaky_relu_forward", "pwgb_tade_combine_forward",
    "pwgb_tade_gate_forward", "pwgb_instance_norm_backward", "pwgb_upsample_nearest_backward", "pwgb_tade_combine_backward",
    "pwgb_tade_gate_backward",
    "pwgb_stft_amplitude_backward", "pwgb_mel_project_backward", "pwgb_gate_forward", "pwgb_gate_backward",
    "pwgb_upsample_fir_backward", "pwgb_stft_loss_terms", "pwgb_stft_loss_dmag",
    "pwgb_symbol_embed_forward", "pwgb_symbol_embed_backward_workspace", "pwgb_symbol_embed_backward",
    "pwgb_channel_layernorm_forward", "pwgb_channel_layernorm_backward_workspace", "pwgb_channel_layernorm_backward",
    "pwgb_duration_loss_forward", "pwgb_duration_loss_backward", "pwgb_duration_round", "pwgb_collate_runlength",
    "pwgb_vq_forward", "pwgb_vq_backward",
]
