"""Tensor-level wrappers over the C ABI (include/pwgb.h).

PyTorch is plumbing here: it owns device memory and the stream.  Every function
checks that its tensors live on a CUDA device and raises otherwise -- there is no
CPU path in this package.
"""
import ctypes as C
import math
import os

import torch

from . import capi
from .capi import ACT_LRELU, ACT_NONE, ACT_TANH, PAD_REFLECT, PAD_REPLICATE, PAD_ZERO, PwgbError

# Optional per-launch instrumentation used by bench.py / profiling (None = off).  When set
# to a list, every wrapper appends (kernel_class, algorithmic_flops, algorithmic_bytes,
# start_event, end_event) recorded on the launching stream.
PROFILE = None


class _Prof:
    __slots__ = ("name", "flops", "bytes", "e0", "desc")

    def __init__(self, name, flops, nbytes, desc=""):
        self.name, self.flops, self.bytes, self.desc = name, flops, nbytes, desc
        self.e0 = None
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def done(self):
        if self.e0 is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.append((self.name, self.flops, self.bytes, self.e0, e1, self.desc))


# Engine selection: "auto" = tensor-core path whenever pwgb_conv1d_tc_supported() says so, else the
# FFMA kernel; "simt" forces the FFMA kernel (used by tests to cross-check the two paths).
ENGINE = os.environ.get("PWGB_ENGINE", "auto")


def packed_weight(w, groups=1):
    """bf16 hi/lo operand image of a conv weight for the tensor-core path, cached on the tensor
    object and invalidated by its version counter (in-place updates) -- a temporary such as a
    weight-norm product is simply re-packed every forward."""
    cache = getattr(w, "_pwgb_packed", None)
    if cache is not None and cache[0] == w._version and cache[1].device == w.device:
        return cache[1]
    cout, cin, K = w.shape  # cin = channels per group
    L = capi.lib()
    nbytes = L.pwgb_conv1d_tc_packed_weight_bytes(cin, cout, K)
    buf = torch.empty(nbytes // 4, device=w.device, dtype=torch.int32)
    rc = L.pwgb_conv1d_tc_pack_weight_grouped(_p(w), cin, cout, K, int(groups), _p(buf), _stream())
    capi.check(rc, "pwgb_conv1d_tc_pack_weight")
    try:
        w._pwgb_packed = (w._version, buf)
    except Exception:
        pass
    return buf


_DESC_CACHE = {}
_PAD = {"zero": PAD_ZERO, "zeros": PAD_ZERO, "reflect": PAD_REFLECT, "replicate": PAD_REPLICATE}
_ACT = {None: ACT_NONE, "none": ACT_NONE, "tanh": ACT_TANH, "lrelu": ACT_LRELU}


def _dev(t, name):
    if not isinstance(t, torch.Tensor):
        raise PwgbError(f"{name}: expected a torch.Tensor")
    if not t.is_cuda:
        raise PwgbError(f"{name}: tensor is on {t.device}; parallelwavegan_b200 only runs on CUDA (no CPU fallback)")
    if t.dtype != torch.float32:
        raise PwgbError(f"{name}: expected float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_cur_device = getattr(torch._C, "_cuda_getDevice", None)


def _stream():
    """The current CUDA stream handle.  torch.cuda.current_stream() builds a Stream object through several Python
    layers (15 us: 20 % of the host time of a training step with ~2000 launches); the raw getter is one C call."""
    if _raw_stream is not None and _cur_device is not None:
        return C.c_void_p(_raw_stream(_cur_device()))
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def conv1d_raw(
    x,
    w,
    bias=None,
    *,
    stride=1,
    padding=0,
    dilation=1,
    groups=1,
    pad_mode="zero",
    pre_slope=1.0,
    pre_gate=False,
    post_act=None,
    post_slope=0.0,
    residual=None,
    out_scale=1.0,
    out=None,
    accumulate=False,
    period=1,
):
    """y = [y +] out_scale * (act(conv(pre(x)) + bias) + residual)   -- pwgb_conv1d_forward.

    ``padding``: int or (left, right) rows.  ``period`` > 1 treats x as the
    (B, C, ceil(L/P), P) view of HiFiGANPeriodDiscriminator (reflect-extended to a
    multiple of P, hifigan.py:365-369) and returns a 4-D tensor."""
    x = _dev(x, "x")
    w = _dev(w, "w")
    if w.dim() == 4:  # Conv2d (k, 1) weights of the period discriminators
        w = w.reshape(w.shape[0], w.shape[1], w.shape[2])
    B, cin_x = x.shape[0], x.shape[1]
    L = math.prod(x.shape[2:])  # from the shape, so that an empty batch keeps its length
    cout, cin_g, K = w.shape
    cin = cin_g * groups
    if cin_x != cin * (2 if pre_gate else 1):
        raise PwgbError(f"conv1d: x has {cin_x} channels, weight expects {cin}")
    P = int(period)
    pl, pr = (padding, padding) if isinstance(padding, int) else padding
    if P > 1 and stride == 1 and L % P == 0 and out is None and residual is None:
        # a (k,1) Conv2d with stride 1 over the (rows, P) view IS a 1-D conv over the flat axis with
        # dilation P and zero padding pad*P (rows outside [0, R) are flat indices outside [0, R*P)):
        # this puts the wide 1024-channel period layers on the tensor-core path
        y = conv1d_raw(x.reshape(B, cin_x, L), w, bias, stride=1, padding=(pl * P, pr * P), dilation=dilation * P, groups=groups,
                       pad_mode=pad_mode, pre_slope=pre_slope, pre_gate=pre_gate, post_act=post_act, post_slope=post_slope,
                       out_scale=out_scale)
        return y.reshape(B, cout, y.shape[-1] // P, P)
    t_in = (L + P - 1) // P
    t_out = (t_in + pl + pr - dilation * (K - 1) - 1) // stride + 1
    if t_out < 0:
        raise PwgbError("conv1d: input shorter than the receptive field")
    shape = (B, cout, t_out) if P == 1 else (B, cout, t_out, P)
    if out is None:
        if accumulate:
            raise PwgbError("conv1d: accumulate needs `out`")
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
    else:
        out = _dev(out, "out")
        if tuple(out.shape) != shape:
            raise PwgbError(f"conv1d: out has shape {tuple(out.shape)}, expected {shape}")
    if residual is not None:
        residual = _dev(residual, "residual")
        if residual.numel() != out.numel():
            raise PwgbError("conv1d: residual shape mismatch")
        if out.numel() and residual.data_ptr() == out.data_ptr():
            raise PwgbError("conv1d: residual must not alias out")
    if out.numel() == 0:
        return out  # an empty batch: nothing to compute (and no device pointers to pass)
    if bias is not None:
        bias = _dev(bias, "bias")
    # descriptors are immutable on the C side: one ctypes object per distinct configuration (building a 25-field
    # Structure costs ~6 us, a training step issues ~750 convolutions)
    dkey = (B, cin, cout, t_in, t_out, K, stride, dilation, groups, pl, pad_mode, P, L, float(pre_slope), bool(pre_gate), post_act,
            float(post_slope), float(out_scale), bool(accumulate))
    d = _DESC_CACHE.get(dkey)
    if d is None:
        if len(_DESC_CACHE) > 4096:
            _DESC_CACHE.clear()
        d = _DESC_CACHE[dkey] = capi.Conv1dDesc(
            batch=B, cin=cin, cout=cout, t_in=t_in, t_out=t_out, kernel=K, stride=stride, dilation=dilation,
            groups=groups, pad_left=pl, pad_mode=_PAD[pad_mode], period=P, t_valid=L, pre_slope=float(pre_slope),
            pre_gate=int(bool(pre_gate)), post_act=_ACT[post_act], post_slope=float(post_slope),
            out_scale=float(out_scale), accumulate=int(bool(accumulate)), shuffle=0, shuffle_pad=0, shuffle_tout=0,
            x_batch_stride=0, y_batch_stride=0, r_batch_stride=0,
        )
    prof = _Prof("conv1d", 2.0 * B * cout * t_out * P * cin_g * K,
                 4.0 * (x.numel() + out.numel() * (2 if accumulate else 1) + (residual.numel() if residual is not None else 0)),
                 f"B{B} cin{cin} cout{cout} k{K} d{dilation} s{stride} g{groups} T{t_out}" if PROFILE is not None else "")
    L = capi.lib()
    if ENGINE != "simt" and L.pwgb_conv1d_tc_supported(C.byref(d)):
        pk = packed_weight(w, groups)
        prof.name = "conv1d_tc"
        rc = L.pwgb_conv1d_tc_forward(C.byref(d), _p(x), _p(pk), _p(bias), _p(residual), _p(out), _stream())
        capi.check(rc, "pwgb_conv1d_tc_forward")
    else:
        rc = L.pwgb_conv1d_forward(C.byref(d), _p(x), _p(w), _p(bias), _p(residual), _p(out), _stream())
        capi.check(rc, "pwgb_conv1d_forward")
    prof.done()
    return out


def resblock_pair(x, w1, b1, w2, b2, *, kernel_size, dilation, slope, out=None, accumulate=False, out_scale=1.0):
    """One HiFi-GAN ResBlock conv pair in one launch (pwgb_resblock_pair_forward), inference only:
        x' = conv_{k,1}(lrelu(conv_{k,d}(lrelu(x)) + b1)) + b2 + x     ("same" zero padding, LeakyReLU ``slope``)
    returned as ``out_scale * x'``, or written / added into ``out``.  Bit-identical to the two conv1d calls it replaces.
    Returns None when the fused kernel does not serve the call (autograd, the FFMA engine, channel counts other than
    32 / 64, t % 4 != 0, unaligned tensors): the caller then runs the two convs."""
    if ENGINE == "simt" or _needs_grad(x, w1, b1, w2, b2):
        return None
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.is_contiguous()):
        return None
    B, Cc, T = x.shape
    K = int(kernel_size)
    if tuple(w1.shape) != (Cc, Cc, K) or tuple(w2.shape) != (Cc, Cc, K) or x.data_ptr() % 16:
        return None
    if out is not None and (tuple(out.shape) != tuple(x.shape) or not out.is_contiguous() or out.dtype != torch.float32
                            or out.data_ptr() % 16 or out.data_ptr() == x.data_ptr()):
        return None
    if accumulate and out is None:
        raise PwgbError("resblock_pair: accumulate needs `out`")
    dkey = ("resblock", B, Cc, T, K, int(dilation), float(slope), float(out_scale), bool(accumulate))
    d = _DESC_CACHE.get(dkey)
    if d is None:
        if len(_DESC_CACHE) > 4096:
            _DESC_CACHE.clear()
        d = _DESC_CACHE[dkey] = capi.ResBlockDesc(batch=B, channels=Cc, t=T, kernel=K, dilation=int(dilation), slope=float(slope),
                                                  out_scale=float(out_scale), accumulate=int(bool(accumulate)))
    L = capi.lib()
    if not L.pwgb_resblock_pair_supported(C.byref(d)):
        return None
    w1, w2 = _dev(w1, "w1"), _dev(w2, "w2")
    b1 = _dev(b1, "b1") if b1 is not None else None
    b2 = _dev(b2, "b2") if b2 is not None else None
    if out is None:
        out = torch.empty_like(x)
    if out.numel() == 0:
        return out  # an empty batch: nothing to compute (and no device pointers to pass)
    pk1, pk2 = packed_weight(w1), packed_weight(w2)
    # FLOPs of both convs; bytes: x once, out written (and read too when accumulating), the intermediate stays on chip
    prof = _Prof("resblock_pair_tc", 2 * 2.0 * B * Cc * T * Cc * K, 4.0 * (x.numel() + out.numel() * (2 if accumulate else 1)),
                 f"B{B} C{Cc} k{K} d{dilation} T{T}" if PROFILE is not None else "")
    rc = L.pwgb_resblock_pair_forward(C.byref(d), _p(x), _p(pk1), _p(b1), _p(pk2), _p(b2), _p(out), _stream())
    capi.check(rc, "pwgb_resblock_pair_forward")
    prof.done()
    return out


def resblock_pair_plan(channels, t, kernel_size, dilation, batch=1):
    """The fused pair's tile plan as a dict (output rows per tile, conv rows per tile, conv1 operand buffers, weight
    stages of both rings, raw activation stages, and the kernel: "split" = one consumer warpgroup per conv, "lockstep" =
    both warpgroups through both convs), or None when the pair keeps the two-launch path."""
    d = capi.ResBlockDesc(batch=batch, channels=channels, t=t, kernel=kernel_size, dilation=dilation, slope=0.1, out_scale=1.0,
                          accumulate=0)
    L = capi.lib()
    v = (C.c_int * 5)()
    if not L.pwgb_resblock_pair_plan(C.byref(d), v):
        return None
    plan = dict(zip(("M2", "TT", "na", "nb", "ns"), list(v)))
    plan["variant"] = {1: "lockstep", 2: "split"}[L.pwgb_resblock_pair_variant(C.byref(d))]
    return plan


def conv_transpose1d_raw(x, w, bias=None, *, stride, padding=0, output_padding=0, pre_slope=1.0, groups=1, period=1):
    """ConvTranspose1d with fused pre-LeakyReLU -- pwgb_conv_transpose1d_forward.
    w is the reference layout (cin, cout, k)."""
    x = _dev(x, "x")
    w = _dev(w, "w")
    if w.dim() == 4:
        w = w.reshape(w.shape[0], w.shape[1], w.shape[2])
    B, cin = x.shape[0], x.shape[1]
    P = int(period)
    t_in = math.prod(x.shape[2:]) // P
    if w.shape[0] != cin:
        raise PwgbError(f"conv_transpose1d: x has {cin} channels, weight expects {w.shape[0]}")
    cout, K = w.shape[1] * groups, w.shape[2]
    t_out = (t_in - 1) * stride - 2 * padding + K + output_padding
    if bias is not None:
        bias = _dev(bias, "bias")
    d = capi.ConvTr1dDesc(batch=B, cin=cin, cout=cout, t_in=t_in, t_out=t_out, kernel=K, stride=stride,
                          padding=padding, pre_slope=float(pre_slope), groups=int(groups), period=P)
    L = capi.lib()
    nbytes = L.pwgb_conv_transpose1d_workspace(C.byref(d))
    ws = torch.empty((nbytes + 3) // 4, device=x.device, dtype=torch.float32)
    y = torch.empty((B, cout, t_out) if P == 1 else (B, cout, t_out, P), device=x.device, dtype=torch.float32)
    if y.numel() == 0:
        return y  # an empty batch: nothing to compute
    prof = _Prof("conv_transpose1d", 2.0 * B * cout * t_out * cin * ((K + stride - 1) // stride), 4.0 * (x.numel() + y.numel()),
                 f"B{B} cin{cin} cout{cout} k{K} s{stride} T{t_out}")
    rc = L.pwgb_conv_transpose1d_forward(C.byref(d), _p(x), _p(w), _p(bias), _p(y), _p(ws), C.c_size_t(nbytes), _stream())
    capi.check(rc, "pwgb_conv_transpose1d_forward")
    prof.done()
    return y


def conv_transpose1d_cat_raw(x1, x2, w, bias=None, *, stride, padding=0, output_padding=0, pre_slope=1.0):
    """conv_transpose1d_raw on torch.cat((x1, x2), dim=1) -- pwgb_conv_transpose1d_cat_forward, which reads the two
    sources in place, bit-identical to the single-source entry on the concatenation.  Configurations it does not serve
    (x1's channels not a multiple of 32, the FFMA conv-transpose) concatenate and call the single-source entry."""
    x1, x2, w = _dev(x1, "x1"), _dev(x2, "x2"), _dev(w, "w")
    B, cin1, t_in = x1.shape
    if x2.dim() != 3 or x2.shape[0] != B or x2.shape[2] != t_in:
        raise PwgbError(f"conv_transpose1d_cat: x1 {tuple(x1.shape)} and x2 {tuple(x2.shape)} do not concatenate along channels")
    cin = cin1 + x2.shape[1]
    if w.shape[0] != cin:
        raise PwgbError(f"conv_transpose1d_cat: inputs have {cin} channels, weight expects {w.shape[0]}")
    cout, K = w.shape[1], w.shape[2]
    t_out = (t_in - 1) * stride - 2 * padding + K + output_padding
    d = capi.ConvTr1dDesc(batch=B, cin=cin, cout=cout, t_in=t_in, t_out=t_out, kernel=K, stride=stride, padding=padding,
                          pre_slope=float(pre_slope), groups=1, period=1)
    L = capi.lib()
    if ENGINE == "simt" or not L.pwgb_conv_transpose1d_cat_supported(C.byref(d), cin1):
        return conv_transpose1d_raw(torch.cat((x1, x2), dim=1), w, bias, stride=stride, padding=padding,
                                    output_padding=output_padding, pre_slope=pre_slope)
    if bias is not None:
        bias = _dev(bias, "bias")
    nbytes = L.pwgb_conv_transpose1d_workspace(C.byref(d))
    ws = torch.empty((nbytes + 3) // 4, device=x1.device, dtype=torch.float32)
    y = torch.empty((B, cout, t_out), device=x1.device, dtype=torch.float32)
    if y.numel() == 0:
        return y  # an empty batch: nothing to compute
    prof = _Prof("conv_transpose1d_cat", 2.0 * B * cout * t_out * cin * ((K + stride - 1) // stride),
                 4.0 * (x1.numel() + x2.numel() + y.numel()), f"B{B} cin{cin1}+{cin - cin1} cout{cout} k{K} s{stride} T{t_out}")
    rc = L.pwgb_conv_transpose1d_cat_forward(C.byref(d), cin1, _p(x1), _p(x2), _p(w), _p(bias), _p(y), _p(ws),
                                             C.c_size_t(nbytes), _stream())
    capi.check(rc, "pwgb_conv_transpose1d_cat_forward")
    prof.done()
    return y


def dropout_raw(x, p, seed, offset=0, backward=False):
    """Training-mode dropout with the counter-based mask of (seed, offset) -- pwgb_dropout_forward; ``backward``
    applies the same mask and scale to a gradient (pwgb_dropout_backward)."""
    x = _dev(x, "x")
    y = torch.empty_like(x)
    fn = capi.lib().pwgb_dropout_backward if backward else capi.lib().pwgb_dropout_forward
    rc = fn(_p(x) if x.numel() else None, _p(y) if y.numel() else None, x.numel(), float(p), int(seed), int(offset), _stream())
    capi.check(rc, "pwgb_dropout_backward" if backward else "pwgb_dropout_forward")
    return y


def dropout(x, p, training):
    """torch.nn.Dropout(p) semantics: identity (no launch) in eval mode or at p == 0, else a fresh mask per call whose
    seed is drawn from torch's default CPU generator -- no device sync, and ``torch.manual_seed`` makes it
    reproducible.  Applied in training mode also under ``no_grad`` (the discriminator phase regenerates the
    generator's output under no_grad with the generator still in train())."""
    if not training or p == 0:
        return x
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    if _needs_grad(x):
        from . import autograd as ag

        return ag.DropoutFn.apply(x, float(p), seed)
    return dropout_raw(x, p, seed)


def upsample_fir(x, fir, scale, out=None, out_channels=None):
    """One stage of the PWG conditioning upsampler (layers/upsample.py:112-128):
    nearest repeat x`scale` + (2*scale+1)-tap FIR, zero padded -- pwgb_upsample_fir_forward.
    x: (B, C, T) -> (B, C, T*scale); with ``out_channels`` > C the result is written into the
    first C channels of a zero-initialised (B, out_channels, T*scale) tensor (channel padding
    for the tensor-core conditioning contraction)."""
    x = _dev(x, "x")
    fir = _dev(fir, "fir").reshape(-1)
    B, Cc, T = x.shape
    if fir.numel() != 2 * scale + 1:
        raise PwgbError("upsample_fir: filter must have 2*scale+1 taps")
    oc = Cc if out_channels is None else int(out_channels)
    if out is None:
        out = (torch.zeros if oc != Cc else torch.empty)((B, oc, T * scale), device=x.device, dtype=torch.float32)
    prof = _Prof("upsample_fir", 2.0 * B * Cc * T * scale * (2 * scale + 1), 4.0 * (x.numel() + B * Cc * T * scale), f"B{B} C{Cc} T{T} s{scale}")
    rc = capi.lib().pwgb_upsample_fir_forward(B * Cc, Cc, T, int(scale), _p(x), _p(fir), _p(out), oc * T * scale, _stream())
    capi.check(rc, "pwgb_upsample_fir_forward")
    prof.done()
    return out


class WaveNetLayerWeights:
    """Device-side operand images of one WaveNetResidualBlock for pwgb_wavenet_layer_forward."""

    __slots__ = ("desc", "packed", "b_conv", "b_skip_out", "key")


def param_key(*mods):
    """Cache key for data derived from module parameters: identity and version counter of every LEAF
    parameter / buffer (weight_g, weight_v, weight, bias ...).  Effective weights are temporaries under
    weight norm (fresh tensor, version 0, recycled address), so they must never be the key.  In-place
    updates through ``.data`` do not bump the version counter: call ``invalidate_caches(module)`` after
    such surgery."""
    key = []
    for m in mods:
        if m is None:
            continue
        for t in list(m.parameters(recurse=False)) + list(m.buffers(recurse=False)):
            key.append((id(t), t._version, t.data_ptr()))
    return tuple(key)


def invalidate_caches(module):
    """Drop every packed-operand cache below ``module`` (after weight surgery through ``.data``)."""
    for m in module.modules():
        c = getattr(m, "_cache", None)
        if isinstance(c, dict):
            c.clear()
        for t in list(m.parameters(recurse=False)):
            if hasattr(t, "_pwgb_packed"):
                try:
                    del t._pwgb_packed
                except Exception:
                    pass


def wavenet_layer(x, c, w_conv, b_conv, w_aux, w_skip, b_skip, w_out, b_out, dilation, skips, aux_real, cache=None, key=None):
    """WaveNetResidualBlock.forward (layers/residual_block.py:102-140), in place on ``skips``:
    returns x_out.  ``c``: (B, aux_pad, T) conditioning, zero-padded to a multiple of 32 channels
    (or None).  Uses the fused tensor-core layer when pwgb_wavenet_supported(), otherwise composes the
    layer from the generic fused conv (gate pre-op, accumulate, residual epilogue)."""
    x = _dev(x, "x")
    B, R, T = x.shape
    G, _, K = w_conv.shape
    S = w_skip.shape[0]
    L = capi.lib()
    aux_pad = 0 if c is None else c.shape[1]
    d = capi.WaveNetDesc(batch=B, t=T, residual_channels=R, gate_channels=G, skip_channels=S, aux_channels=aux_pad,
                         kernel=K, dilation=int(dilation))
    if ENGINE != "simt" and L.pwgb_wavenet_supported(C.byref(d)):
        # ``key`` identifies the leaf parameters the effective weights were derived from (param_key); without
        # it nothing is cached (effective weights are temporaries whose address / version say nothing)
        ent = cache.get("wn") if (cache is not None and key is not None) else None
        if ent is None or ent[0] != key:
            nbytes = L.pwgb_wavenet_packed_bytes(C.byref(d))
            packed = torch.empty(nbytes // 4, device=x.device, dtype=torch.int32)
            rc = L.pwgb_wavenet_pack(C.byref(d), _p(_dev(w_conv, "w_conv")), _p(w_aux.contiguous() if w_aux is not None else None),
                                     int(aux_real), _p(_dev(w_skip, "w_skip")), _p(_dev(w_out, "w_out")), _p(packed), _stream())
            capi.check(rc, "pwgb_wavenet_pack")
            bso = None
            if b_skip is not None:
                bso = torch.cat([b_skip.detach().reshape(-1), b_out.detach().reshape(-1)]).contiguous()
            ent = (key, packed, bso)
            if cache is not None and key is not None:
                cache["wn"] = ent
        _, packed, bso = ent
        g_ws = torch.empty((B, G, T), device=x.device, dtype=torch.float32)
        x_out = torch.empty_like(x)
        prof = _Prof("wavenet_layer_tc", 2.0 * B * T * (G * R * K + G * aux_real + (S + R) * (G // 2)),
                     4.0 * B * T * (2 * R + aux_real + 2 * S), f"B{B} R{R} G{G} S{S} A{aux_real} k{K} d{dilation} T{T}")
        rc = L.pwgb_wavenet_layer_forward(C.byref(d), _p(x), _p(c), _p(packed), _p(b_conv), _p(bso), _p(x_out), _p(skips), _p(g_ws), _stream())
        capi.check(rc, "pwgb_wavenet_layer_forward")
        prof.done()
        return x_out
    # generic composition (any channel counts): 4 launches
    g = conv1d(x, w_conv, b_conv, dilation=dilation, padding=(K - 1) // 2 * dilation)
    if c is not None:
        wa = w_aux
        if c.shape[1] != w_aux.shape[1]:  # conditioning stored channel-padded
            wa = torch.nn.functional.pad(w_aux, (0, 0, 0, c.shape[1] - w_aux.shape[1]))
        conv1d(c, wa, None, out=g, accumulate=True)
    conv1d(g, w_skip, b_skip, pre_gate=True, out=skips, accumulate=True)
    return conv1d(g, w_out, b_out, pre_gate=True, residual=x, out_scale=0.7071067811865476)


class WnStack:
    """Packed WaveNet residual stack (pwgb_wnstack_*): the residual stream and the conditioning stay in the
    tensor core's operand layout (bf16 hi/lo) between the fused one-kernel layers.  Holds the two ping-pong
    stream buffers (zero halos, allocated once per (B, T)) and the packed conditioning."""

    def __init__(self, B, T, R, G, S, A, K, max_dilation, device):
        self.desc = capi.WnStackDesc(batch=B, t=T, residual_channels=R, gate_channels=G, skip_channels=S, aux_channels=A,
                                     kernel=K, halo=(K - 1) // 2 * int(max_dilation))
        L = capi.lib()
        if not L.pwgb_wnstack_supported(C.byref(self.desc)):
            raise PwgbError("wnstack: configuration not supported by the fused tensor-core layer")
        nx = L.pwgb_wnstack_x_bytes(C.byref(self.desc))
        nc = L.pwgb_wnstack_c_bytes(C.byref(self.desc))
        self.x = [torch.zeros(nx // 4, device=device, dtype=torch.int32) for _ in range(2)]  # zero halos: written once
        self.c = torch.empty(nc // 4, device=device, dtype=torch.int32)
        self.cur = 0
        self.shape = (B, R, T)
        self.S, self.A = S, A

    @staticmethod
    def supported(B, T, R, G, S, A, K, max_dilation):
        d = capi.WnStackDesc(batch=B, t=T, residual_channels=R, gate_channels=G, skip_channels=S, aux_channels=A, kernel=K,
                             halo=(K - 1) // 2 * int(max_dilation))
        return ENGINE != "simt" and bool(capi.lib().pwgb_wnstack_supported(C.byref(d)))

    def pack_c(self, c):
        """c: (B, >= A, T) fp32 conditioning at the waveform rate."""
        c = _dev(c, "c")
        B, Cs, T = c.shape
        if (B, T) != (self.shape[0], self.shape[2]) or Cs < self.A:
            raise PwgbError(f"wnstack.pack_c: conditioning shape {tuple(c.shape)} does not match the stack")
        prof = _Prof("wn_pack_c", 0.0, 8.0 * B * self.A * T, f"B{B} A{self.A} T{T}")
        rc = capi.lib().pwgb_wnstack_pack_c(C.byref(self.desc), _p(c), Cs * T, _p(self.c), _stream())
        capi.check(rc, "pwgb_wnstack_pack_c")
        prof.done()

    def pack_x(self, x):
        x = _dev(x, "x")
        if tuple(x.shape) != self.shape:
            raise PwgbError(f"wnstack.pack_x: expected {self.shape}, got {tuple(x.shape)}")
        rc = capi.lib().pwgb_wnstack_pack_x(C.byref(self.desc), _p(x), _p(self.x[self.cur]), _stream())
        capi.check(rc, "pwgb_wnstack_pack_x")

    def unpack_x(self):
        x = torch.empty(self.shape, device=self.c.device, dtype=torch.float32)
        rc = capi.lib().pwgb_wnstack_unpack_x(C.byref(self.desc), _p(self.x[self.cur]), _p(x), _stream())
        capi.check(rc, "pwgb_wnstack_unpack_x")
        return x

    def first_conv(self, z, w, bias):
        """Conv1d1x1 in_channels -> R on the noise, written straight into the packed stream."""
        z = _dev(z, "z")
        w = _dev(w, "w").reshape(w.shape[0], -1)
        B, cin, T = z.shape
        if (B, T) != (self.shape[0], self.shape[2]) or w.shape != (self.shape[1], cin):
            raise PwgbError("wnstack.first_conv: shape mismatch")
        prof = _Prof("wn_first_conv", 2.0 * B * T * cin * self.shape[1], 4.0 * B * T * (cin + self.shape[1]), f"B{B} T{T}")
        rc = capi.lib().pwgb_wnstack_first_conv(C.byref(self.desc), _p(z), cin, _p(w), _p(bias), _p(self.x[self.cur]), _stream())
        capi.check(rc, "pwgb_wnstack_first_conv")
        prof.done()

    def layer(self, packed, b_conv, b_skip_out, dilation, skips, skips_init=False, write_x=True):
        """One fused layer on the current stream buffer; the result becomes the current buffer."""
        B, R, T = self.shape
        G = self.desc.gate_channels
        K = self.desc.kernel
        prof = _Prof("wavenet_fused_tc", 2.0 * B * T * (G * R * K + G * self.A + (self.S + R) * (G // 2)),
                     4.0 * B * T * ((2 if write_x else 1) * R + self.A + (1 if skips_init else 2) * self.S),
                     f"B{B} R{R} G{G} S{self.S} A{self.A} k{K} d{dilation} T{T}")
        nxt = self.x[1 - self.cur] if write_x else None
        rc = capi.lib().pwgb_wnstack_layer_forward(C.byref(self.desc), int(dilation), _p(self.x[self.cur]), _p(self.c), _p(packed),
                                                   _p(b_conv), _p(b_skip_out), _p(nxt), _p(skips), int(bool(skips_init)), _stream())
        capi.check(rc, "pwgb_wnstack_layer_forward")
        prof.done()
        if write_x:
            self.cur = 1 - self.cur


def wavenet_packed_weights(w_conv, w_aux, w_skip, w_out, b_skip, b_out, aux_real, cache=None, key=None):
    """Operand images of one WaveNet layer (pwgb_wavenet_pack, conditioning weight padded to a multiple of 32
    input channels) + concat(b_skip, b_out); cached under ``key`` (see param_key)."""
    ent = cache.get("wnp") if (cache is not None and key is not None) else None
    if ent is not None and ent[0] == key:
        return ent[1], ent[2]
    G, R, K = w_conv.shape
    S = w_skip.shape[0]
    aux_pad = (aux_real + 31) // 32 * 32
    d = capi.WaveNetDesc(batch=1, t=128, residual_channels=R, gate_channels=G, skip_channels=S, aux_channels=aux_pad, kernel=K, dilation=1)
    L = capi.lib()
    nbytes = L.pwgb_wavenet_packed_bytes(C.byref(d))
    if nbytes == 0:
        raise PwgbError("wavenet_packed_weights: configuration not supported")
    packed = torch.empty(nbytes // 4, device=w_conv.device, dtype=torch.int32)
    rc = L.pwgb_wavenet_pack(C.byref(d), _p(_dev(w_conv, "w_conv")), _p(_dev(w_aux, "w_aux").reshape(G, -1).contiguous()), int(aux_real),
                             _p(_dev(w_skip, "w_skip")), _p(_dev(w_out, "w_out")), _p(packed), _stream())
    capi.check(rc, "pwgb_wavenet_pack")
    bso = None
    if b_skip is not None:
        bso = torch.cat([b_skip.detach().reshape(-1), b_out.detach().reshape(-1)]).contiguous()
    if cache is not None and key is not None:
        cache["wnp"] = (key, packed, bso)
    return packed, bso


def mr_stft_loss(x, y, fft_sizes, hop_sizes, win_lengths, windows, eps=1e-7):
    """MultiResolutionSTFTLoss.forward (losses/stft_loss.py:146-170) -> device tensor [sc, mag].
    x, y: (B, T) or (B, C, T); windows: list of device tensors (win_length,)."""
    x = _dev(x, "x")
    y = _dev(y, "y")
    if x.dim() == 3:
        x = x.reshape(-1, x.shape[2])
        y = y.reshape(-1, y.shape[2])
    if x.shape != y.shape:
        raise PwgbError("mr_stft_loss: x and y must have the same shape")
    B, T = x.shape
    n = len(fft_sizes)
    descs = (capi.StftDesc * n)(*[capi.StftDesc(batch=B, t=T, n_fft=int(f), hop=int(h), win_length=int(w), clamp_eps=float(eps))
                                  for f, h, w in zip(fft_sizes, hop_sizes, win_lengths)])
    wins = [_dev(w, "window") for w in windows]
    wptr = (C.c_void_p * n)(*[w.data_ptr() for w in wins])
    L = capi.lib()
    nbytes = L.pwgb_mr_stft_loss_workspace(descs, n)
    if nbytes == 0:
        raise PwgbError("mr_stft_loss: unsupported STFT configuration (n_fft must be a power of two <= 4096 and T > n_fft/2)")
    ws = torch.empty((nbytes + 3) // 4, device=x.device, dtype=torch.float32)
    out = torch.empty(2, device=x.device, dtype=torch.float32)
    prof = _Prof("mr_stft_loss", 0.0, 8.0 * B * T, f"B{B} T{T} res{n}")
    rc = L.pwgb_mr_stft_loss_forward(descs, n, _p(x), _p(y), wptr, _p(out), _p(ws), C.c_size_t(nbytes), _stream())
    capi.check(rc, "pwgb_mr_stft_loss_forward")
    prof.done()
    return out


def stft_amplitude(x, y, n_fft, hop, win_length, window, eps):
    """sqrt(clamp(|STFT|^2, eps)) as (B, frames, bins) for x and (optionally) y."""
    x = _dev(x, "x")
    B, T = x.shape
    d = capi.StftDesc(batch=B, t=T, n_fft=int(n_fft), hop=int(hop), win_length=int(win_length), clamp_eps=float(eps))
    frames, bins = 1 + T // hop, n_fft // 2 + 1
    ax = torch.empty((B, frames, bins), device=x.device, dtype=torch.float32)
    ay = None
    if y is not None:
        y = _dev(y, "y")
        ay = torch.empty_like(ax)
    rc = capi.lib().pwgb_stft_amplitude_forward(C.byref(d), _p(x), _p(y), _p(_dev(window, "window")), _p(ax), _p(ay), _stream())
    capi.check(rc, "pwgb_stft_amplitude_forward")
    return ax, ay


def mel_project(ax, ay, melmat, eps, log_scale, want_mel=True, want_loss=False):
    """clamp(amp @ melmat, eps) -> log * log_scale; returns (log-mel of x as (B, n_mels, frames) or None,
    mean-L1 loss between the two log-mels as a 1-element tensor or None)."""
    B, frames, bins = ax.shape
    melmat = _dev(melmat, "melmat")
    n_mels = melmat.shape[1]
    mel = torch.empty((B, n_mels, frames), device=ax.device, dtype=torch.float32) if want_mel else None
    loss = ws = None
    if want_loss:
        loss = torch.empty(1, device=ax.device, dtype=torch.float32)
        ws = torch.empty(B * frames, device=ax.device, dtype=torch.float32)
    rc = capi.lib().pwgb_mel_project_forward(B, frames, bins, n_mels, _p(ax), _p(ay), _p(melmat), float(eps), float(log_scale),
                                             _p(mel), _p(loss), _p(ws), _stream())
    capi.check(rc, "pwgb_mel_project_forward")
    return mel, loss


_REDUCE = {"mse_const": 0, "l1": 1, "hinge": 2, "linear": 3, "mse": 4}


def reduce_mean_raw(mode, x, y=None, c=0.0, s=1.0, weight=1.0, out=None, accumulate=False):
    """out[0] (+)= weight * mean(f(x[, y])) -- pwgb_reduce_mean_forward (deterministic)."""
    x = _dev(x, "x")
    if y is not None:
        y = _dev(y, "y")
        if y.numel() != x.numel():
            raise PwgbError("reduce_mean: size mismatch")
    if out is None:
        out = torch.zeros(1, device=x.device, dtype=torch.float32)
        accumulate = False
    ws = torch.empty(1024, device=x.device, dtype=torch.float32)
    rc = capi.lib().pwgb_reduce_mean_forward(_REDUCE[mode], _p(x), _p(y), x.numel(), float(c), float(s), float(weight),
                                             int(bool(accumulate)), _p(out), _p(ws), 1024, _stream())
    capi.check(rc, "pwgb_reduce_mean_forward")
    return out


def avg_pool1d_raw(x, kernel_size, stride, padding=0, count_include_pad=True):
    """torch.nn.AvgPool1d semantics on (B, C, T) -- pwgb_avg_pool1d_forward."""
    x = _dev(x, "x")
    B, Cc, T = x.shape
    t_out = (T + 2 * padding - kernel_size) // stride + 1
    y = torch.empty((B, Cc, t_out), device=x.device, dtype=torch.float32)
    rc = capi.lib().pwgb_avg_pool1d_forward(_p(x), _p(y), B * Cc, T, int(kernel_size), int(stride), int(padding),
                                            int(bool(count_include_pad)), _stream())
    capi.check(rc, "pwgb_avg_pool1d_forward")
    return y


# --------------------------------------------------------------------------
# backward building blocks (raw wrappers) and autograd-aware public entry points
# --------------------------------------------------------------------------


def conv1d_wgrad(x, gy, w_shape, *, stride=1, padding=0, dilation=1, groups=1, pad_mode="zero", x_slope=1.0, g_slope=1.0, period=1):
    """dw of the conv described by the arguments -- pwgb_conv1d_wgrad (deterministic split reduce)."""
    x = _dev(x, "x")
    gy = _dev(gy, "gy")
    cout, cin_g, K = w_shape[0], w_shape[1], w_shape[2]
    B, cin = x.shape[0], x.shape[1]
    P = int(period)
    L = x.numel() // max(B * cin, 1)
    t_in = (L + P - 1) // P
    t_out = gy.numel() // max(B * cout * P, 1)
    pl = padding if isinstance(padding, int) else padding[0]
    d = capi.Conv1dDesc(batch=B, cin=cin, cout=cout, t_in=t_in, t_out=t_out, kernel=K, stride=stride, dilation=dilation,
                        groups=groups, pad_left=pl, pad_mode=_PAD[pad_mode], period=P, t_valid=L, pre_slope=float(x_slope),
                        out_scale=1.0)
    Lb = capi.lib()
    if P > 1 and stride == 1 and L % P == 0:
        # period conv with stride 1 == dilated 1-D conv over the flat axis (see conv1d_raw)
        return conv1d_wgrad(x.reshape(B, cin, L), gy.reshape(B, cout, -1), w_shape, stride=1, padding=pl * P, dilation=dilation * P,
                            groups=groups, pad_mode=pad_mode, x_slope=x_slope, g_slope=g_slope, period=1)
    if ENGINE != "simt" and Lb.pwgb_conv1d_wgrad_tc_supported(C.byref(d)):
        nbytes = Lb.pwgb_conv1d_wgrad_tc_workspace(C.byref(d))
        ws = torch.empty(max(nbytes // 4, 1), device=x.device, dtype=torch.float32)
        dw = torch.empty((cout, cin_g, K), device=x.device, dtype=torch.float32)
        prof = _Prof("conv1d_wgrad_tc", 2.0 * B * cout * t_out * cin_g * K, 4.0 * (x.numel() + gy.numel()), f"B{B} cin{cin} cout{cout} k{K} d{dilation} T{t_out}")
        rc = Lb.pwgb_conv1d_wgrad_tc(C.byref(d), _p(x), _p(gy), float(g_slope), _p(dw), _p(ws), C.c_size_t(nbytes), _stream())
        capi.check(rc, "pwgb_conv1d_wgrad_tc")
        prof.done()
        return dw
    nbytes = Lb.pwgb_conv1d_wgrad_workspace(C.byref(d))
    ws = torch.empty(max(nbytes // 4, 1), device=x.device, dtype=torch.float32)
    dw = torch.empty((cout, cin_g, K), device=x.device, dtype=torch.float32)
    prof = _Prof("conv1d_wgrad", 2.0 * B * cout * t_out * P * cin_g * K, 4.0 * (x.numel() + gy.numel()), f"B{B} cin{cin} cout{cout} k{K} T{t_out}")
    rc = Lb.pwgb_conv1d_wgrad(C.byref(d), _p(x), _p(gy), float(g_slope), _p(dw), 0, _p(ws), C.c_size_t(nbytes), _stream())
    capi.check(rc, "pwgb_conv1d_wgrad")
    prof.done()
    return dw


def act_backward(mode, g, ref=None, slope=0.0, scale=1.0, out=None, accumulate=False):
    """out (+)= g * scale * f'(ref); mode: "lrelu" (mask ref > 0), "tanh" (ref = output), "scale"."""
    g = _dev(g, "g")
    if ref is not None:
        ref = _dev(ref, "ref")
    if out is None:
        out = torch.empty_like(g)
    rc = capi.lib().pwgb_act_backward({"lrelu": 0, "tanh": 1, "scale": 2}[mode], _p(g), _p(ref), _p(out), g.numel(), float(slope),
                                      float(scale), int(bool(accumulate)), _stream())
    capi.check(rc, "pwgb_act_backward")
    return out


def bias_grad(g, channels):
    g = _dev(g, "g")
    B = g.shape[0]
    db = torch.empty(channels, device=g.device, dtype=torch.float32)
    rc = capi.lib().pwgb_bias_grad(_p(g), _p(db), B, channels, g.numel() // max(B * channels, 1), 0, _stream())
    capi.check(rc, "pwgb_bias_grad")
    return db


def axpby(a, x, b, y):
    """y = a*x + b*y in place on y."""
    x = _dev(x, "x")
    rc = capi.lib().pwgb_axpby(x.numel(), float(a), _p(x), float(b), _p(y), _stream())
    capi.check(rc, "pwgb_axpby")
    return y


# ---- StyleMelGAN glue (forward: raw launches; with gradients: autograd.py Functions over the adjoint kernels) ----
def instance_norm(x, eps=1e-5, pre_slope=1.0):
    """torch.nn.InstanceNorm1d(C) of (B, C, T), optionally on LeakyReLU(x)."""
    x = _dev(x, "x")
    if _needs_grad(x):
        from . import autograd as ag

        return ag.InstanceNormFn.apply(x, float(eps), float(pre_slope))
    B, Cc, T = x.shape
    y = torch.empty_like(x)
    rc = capi.lib().pwgb_instance_norm_forward(_p(x), _p(y), B * Cc, T, float(eps), float(pre_slope), _stream())
    capi.check(rc, "pwgb_instance_norm_forward")
    return y


def upsample_nearest(x, scale):
    """torch.nn.Upsample(scale_factor=scale, mode="nearest") of (B, C, T)."""
    x = _dev(x, "x")
    if scale == 1:
        return x
    if _needs_grad(x):
        from . import autograd as ag

        return ag.UpsampleNearestFn.apply(x, int(scale))
    B, Cc, T = x.shape
    y = torch.empty(B, Cc, T * scale, device=x.device, dtype=torch.float32)
    rc = capi.lib().pwgb_upsample_nearest_forward(_p(x), _p(y), B * Cc, T, int(scale), _stream())
    capi.check(rc, "pwgb_upsample_nearest_forward")
    return y


def leaky_relu(x, slope, inplace=False):
    x = _dev(x, "x")
    if _needs_grad(x):
        from . import autograd as ag

        return ag.LeakyReluFn.apply(x, float(slope))
    y = x if inplace else torch.empty_like(x)
    rc = capi.lib().pwgb_leaky_relu_forward(_p(x), _p(y), x.numel(), float(slope), _stream())
    capi.check(rc, "pwgb_leaky_relu_forward")
    return y


def tade_combine(cg, xn, scale):
    """cg (B, 2C, T), xn (B, C, T / scale) -> cg[:, :C] * nearest(xn, scale) + cg[:, C:]."""
    cg = _dev(cg, "cg")
    xn = _dev(xn, "xn")
    B, C2, T = cg.shape
    Cc = C2 // 2
    if C2 != 2 * Cc or tuple(xn.shape) != (B, Cc, T // scale) or T % scale:
        raise PwgbError(f"tade_combine: shapes {tuple(cg.shape)} / {tuple(xn.shape)} do not match scale {scale}")
    if _needs_grad(cg, xn):
        from . import autograd as ag

        return ag.TadeCombineFn.apply(cg, xn, int(scale))
    y = torch.empty(B, Cc, T, device=cg.device, dtype=torch.float32)
    rc = capi.lib().pwgb_tade_combine_forward(_p(cg), _p(xn), _p(y), B, Cc, T, int(scale), _stream())
    capi.check(rc, "pwgb_tade_combine_forward")
    return y


def tade_gate(x, residual=None, scale=1, gated_function="softmax"):
    """x (B, 2C, T) -> gate(x[:, :C]) * tanh(x[:, C:]) [+ nearest(residual (B, C, T / scale), scale)]."""
    x = _dev(x, "x")
    if gated_function not in ("softmax", "sigmoid"):
        raise PwgbError(f"tade_gate: gated_function={gated_function!r} is not supported")
    B, C2, T = x.shape
    Cc = C2 // 2
    if residual is not None:
        residual = _dev(residual, "residual")
        if tuple(residual.shape) != (B, Cc, T // scale) or T % scale:
            raise PwgbError(f"tade_gate: residual shape {tuple(residual.shape)} does not match {(B, Cc, T // scale)}")
    if _needs_grad(x, residual):
        from . import autograd as ag

        return ag.TadeGateFn.apply(x, residual, int(scale), int(gated_function == "softmax"))
    y = torch.empty(B, Cc, T, device=x.device, dtype=torch.float32)
    rc = capi.lib().pwgb_tade_gate_forward(_p(x), _p(residual), _p(y), B, Cc, T, int(scale), int(gated_function == "softmax"), _stream())
    capi.check(rc, "pwgb_tade_gate_forward")
    return y


def pad1d(x, pad_left, pad_right, mode):
    """Materialised ReflectionPad1d / ReplicationPad1d of (B, C, T) (train-step helper)."""
    x = _dev(x, "x")
    B, Cc, T = x.shape
    xp = torch.empty(B, Cc, T + pad_left + pad_right, device=x.device, dtype=torch.float32)
    rc = capi.lib().pwgb_pad1d_forward(_p(x), _p(xp), B * Cc, T, int(pad_left), int(pad_right), _PAD[mode], _stream())
    capi.check(rc, "pwgb_pad1d_forward")
    return xp


def pad1d_backward(gxp, t, pad_left, pad_right, mode):
    """Adjoint of pad1d: (B, C, pad_left + t + pad_right) -> (B, C, t)."""
    gxp = _dev(gxp, "gxp")
    B, Cc, Te = gxp.shape
    if Te != t + pad_left + pad_right:
        raise PwgbError("pad1d_backward: length mismatch")
    gx = torch.empty(B, Cc, t, device=gxp.device, dtype=torch.float32)
    rc = capi.lib().pwgb_pad1d_backward(_p(gxp), _p(gx), B * Cc, t, int(pad_left), int(pad_right), _PAD[mode], _stream())
    capi.check(rc, "pwgb_pad1d_backward")
    return gx


def _needs_grad(*ts):
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts)


def s2d_raw(x, groups, stride, pad_left, rows_out, period=1, cgo=0):
    """Space-to-depth along time (pwgb_s2d_forward): (B, C, rows[, P]) -> (B, groups*cgo, rows_out[, P]);
    cgo = output channels per group (0: stride * C / groups; larger: zero channels appended per group)."""
    x = _dev(x, "x")
    B, Cc = x.shape[0], x.shape[1]
    P = int(period)
    rows_in = x.numel() // max(B * Cc * P, 1)
    co = groups * cgo if cgo else Cc * stride
    shape = (B, co, rows_out) if P == 1 else (B, co, rows_out, P)
    y = torch.empty(shape, device=x.device, dtype=torch.float32)
    prof = _Prof("s2d", 0.0, 4.0 * (x.numel() + y.numel()), f"B{B} C{Cc} rows{rows_in} P{P} s{stride}")
    rc = capi.lib().pwgb_s2d_forward(_p(x), _p(y), B, Cc, int(groups), rows_in, P, int(stride), int(pad_left), int(rows_out), int(cgo), _stream())
    capi.check(rc, "pwgb_s2d_forward")
    prof.done()
    return y


def s2d_backward_raw(gy, x_shape, groups, stride, pad_left, period=1, cgo=0):
    gy = _dev(gy, "gy")
    B, Cc = x_shape[0], x_shape[1]
    P = int(period)
    n = 1
    for v in x_shape:
        n *= v
    rows_in = n // max(B * Cc * P, 1)
    rows_out = gy.numel() // max(B * (groups * cgo if cgo else Cc * stride) * P, 1)
    gx = torch.empty(x_shape, device=gy.device, dtype=torch.float32)
    rc = capi.lib().pwgb_s2d_backward(_p(gy), _p(gx), B, Cc, int(groups), rows_in, P, int(stride), int(pad_left), int(rows_out), int(cgo), _stream())
    capi.check(rc, "pwgb_s2d_backward")
    return gx


def _conv1d_s2d(x, w, bias, kw):
    """Strided conv on the tensor-core path: space-to-depth + a stride-1 conv with ceil(K/s) taps and s x the
    input channels (pwgb_s2d_forward).  Returns None when the configuration does not qualify.  The weight
    re-layout is torch indexing on the (small) weight tensor, so its backward is autograd's; the activations
    and their gradients only ever pass through libpwgb kernels (s2d / conv / dgrad / wgrad, all stride 1)."""
    stride = int(kw.get("stride", 1))
    if stride <= 1 or ENGINE == "simt" or kw.get("dilation", 1) != 1 or kw.get("pad_mode", "zero") not in ("zero", "zeros"):
        return None
    if kw.get("pre_gate") or kw.get("out") is not None or kw.get("accumulate") or kw.get("residual") is not None:
        return None
    groups, P = int(kw.get("groups", 1)), int(kw.get("period", 1))
    wd = w.shape
    cout, cin_g, K = wd[0], wd[1], wd[2]
    cgo = (cin_g * stride + 31) // 32 * 32  # channels per group after the re-layout, padded to the tensor cores' 32
    if (cout // groups) % 16 or x.dim() < 3 or cgo > 2 * cin_g * stride:
        return None
    if cgo != cin_g * stride and _needs_grad(x, w):
        # zero-padded groups only pay off in the forward: their data / weight gradients have 16-channel groups, which
        # stay on the FFMA kernels -- and those would then work on twice the channels (measured: 3.9 vs 2.1 ms wgrad)
        return None
    B, cin = x.shape[0], x.shape[1]
    L = x.numel() // max(B * cin, 1)
    if L % P or cin != cin_g * groups:
        return None
    rows_in = L // P
    padding = kw.get("padding", 0)
    pl, pr = (padding, padding) if isinstance(padding, int) else padding
    t_out = (rows_in + pl + pr - (K - 1) - 1) // stride + 1
    if t_out <= 0:
        return None
    Kp = (K + stride - 1) // stride
    rows_out = t_out + Kp - 1
    w3 = w.reshape(cout, cin_g, K)
    if Kp * stride != K:
        w3 = torch.nn.functional.pad(w3, (0, Kp * stride - K))
    w2 = w3.reshape(cout, cin_g, Kp, stride).permute(0, 3, 1, 2).reshape(cout, stride * cin_g, Kp)
    if cgo != stride * cin_g:  # zero weight columns for the zero channels the re-layout appends to every group
        w2 = torch.nn.functional.pad(w2, (0, 0, 0, cgo - stride * cin_g))
    if w.dim() == 4:
        w2 = w2.unsqueeze(-1)
    if _needs_grad(x):
        from . import autograd as ag

        xs = ag.S2DFn.apply(x, groups, stride, pl, rows_out, P, cgo)
    else:
        xs = s2d_raw(x, groups, stride, pl, rows_out, P, cgo)
    inner = {k: v for k, v in kw.items() if k not in ("stride", "padding")}
    return conv1d(xs, w2.contiguous(), bias, stride=1, padding=0, **inner)


def _conv1d_padcin(x, w, bias, kw):
    """Input convs on mel features (80 -> 512 k7 of HiFi-GAN, 80 -> 384 of MelGAN): 80 input channels are not a
    multiple of the tensor cores' 32-channel chunk, so the features and the weight are zero-padded to 96 channels (a
    copy of the small (B, 80, frames) tensor) and the conv runs on the tensor-core path instead of the FFMA kernel
    (0.06 vs 0.26 ms at the C2 batch).  Zero channels contribute exact zeros; reflect / replicate padding, activations
    and gradients are unaffected (the pad is torch indexing, differentiable by autograd)."""
    cout, cin_g = w.shape[0], w.shape[1]
    if ENGINE == "simt" or cin_g % 32 == 0 or cin_g < 48 or cout % 16 or kw.get("groups", 1) != 1 or kw.get("stride", 1) != 1:
        return None
    if kw.get("pre_gate") or kw.get("period", 1) != 1 or x.dim() != 3 or w.dim() != 3 or x.shape[1] != cin_g:
        return None
    padc = (cin_g + 31) // 32 * 32 - cin_g
    xp = torch.nn.functional.pad(x, (0, 0, 0, padc))
    wp = torch.nn.functional.pad(w, (0, 0, 0, padc))
    return conv1d(xp, wp, bias, **kw)


def _conv1d_fewcout(x, w, bias, kw):
    """Logit convs of the discriminator towers (1024 -> 1, k3 / (3,1)): wide input, a single output channel.  The weight
    is zero-padded to 16 output channels so that the contraction runs on the tensor cores (N = 16), and channel 0 of the
    result is returned; the padding / slicing are torch indexing on small tensors (differentiable by autograd)."""
    cout, cin_g = w.shape[0], w.shape[1]
    if ENGINE == "simt" or cout >= 16 or cin_g < 256 or cin_g % 32 or kw.get("groups", 1) != 1 or kw.get("stride", 1) != 1:
        return None
    if kw.get("out") is not None or kw.get("accumulate") or kw.get("residual") is not None or kw.get("pre_gate"):
        return None
    if kw.get("pad_mode", "zero") not in ("zero", "zeros"):
        return None
    pad = [0, 0] * (w.dim() - 1) + [0, 16 - cout]
    w16 = torch.nn.functional.pad(w, pad)
    b16 = torch.nn.functional.pad(bias, (0, 16 - cout)) if bias is not None else None
    y = conv1d(x, w16, b16, **kw)
    return y[:, :cout].contiguous()


def conv1d(x, w, bias=None, **kw):
    """Fused conv (see conv1d_raw); differentiable through libpwgb backward kernels when any input requires grad."""
    if kw.get("stride", 1) > 1:
        y = _conv1d_s2d(x, w, bias, kw)
        if y is not None:
            return y
    y = _conv1d_fewcout(x, w, bias, kw)
    if y is not None:
        return y
    y = _conv1d_padcin(x, w, bias, kw)
    if y is not None:
        return y
    if _needs_grad(x, w, bias, kw.get("residual")):
        from . import autograd as ag

        return ag.conv1d(x, w, bias, **kw)
    return conv1d_raw(x, w, bias, **kw)


def conv_transpose1d(x, w, bias=None, **kw):
    if _needs_grad(x, w, bias):
        from . import autograd as ag

        return ag.conv_transpose1d(x, w, bias, **kw)
    return conv_transpose1d_raw(x, w, bias, **kw)


def conv_transpose1d_cat(x1, x2, w, bias=None, **kw):
    """conv_transpose1d on torch.cat((x1, x2), dim=1) without the concatenation (see conv_transpose1d_cat_raw)."""
    if _needs_grad(x1, x2, w, bias):
        from . import autograd as ag

        return ag.conv_transpose1d_cat(x1, x2, w, bias, **kw)
    return conv_transpose1d_cat_raw(x1, x2, w, bias, **kw)


def avg_pool1d(x, kernel_size, stride, padding=0, count_include_pad=True):
    if _needs_grad(x):
        from . import autograd as ag

        return ag.AvgPool1dFn.apply(x, kernel_size, stride, padding, count_include_pad)
    return avg_pool1d_raw(x, kernel_size, stride, padding, count_include_pad)


def reduce_mean(mode, x, y=None, c=0.0, s=1.0, weight=1.0, out=None, accumulate=False):
    if _needs_grad(x, y):
        from . import autograd as ag

        term = ag.ReduceMeanFn.apply(x, y, mode, float(c), float(s), float(weight))
        return term if (out is None or not accumulate) else out + term
    return reduce_mean_raw(mode, x, y, c, s, weight, out, accumulate)


# ---- discrete-symbol front end (models/hifigan.py:867-1289): embedding + length regulation, LayerNorm over channels,
# duration loss and rounding -- pwgb_symbol_embed_* / pwgb_channel_layernorm_* / pwgb_duration_* ----
def _index_tensor(c, name="c"):
    """A (B, K, S) symbol-index tensor read in place by the embed kernels: float32 (the mel2wav collater's features) or
    int64 (the duration collater's codes); any other dtype is cast with ``.long()``, as the reference reads ``c.long()``."""
    if not isinstance(c, torch.Tensor) or not c.is_cuda:
        raise PwgbError(f"{name}: expected a CUDA tensor; parallelwavegan_b200 only runs on CUDA (no CPU fallback)")
    if c.dim() != 3:
        raise PwgbError(f"{name}: expected (B, K, S) indices, got shape {tuple(c.shape)}")
    if c.dtype not in (torch.float32, torch.int64):
        c = c.long()
    return c, int(c.dtype == torch.int64)


def _durations(ds, B, S):
    if not isinstance(ds, torch.Tensor) or not ds.is_cuda or ds.dtype != torch.int64 or tuple(ds.shape) != (B, S):
        raise PwgbError(f"durations: expected a CUDA int64 tensor of shape {(B, S)}")
    if not ds.is_contiguous():
        raise PwgbError("durations: expected a contiguous tensor")
    return ds


def symbol_embed_raw(c, table, spk_table=None, ds=None, t_out=None):
    """(B, C, t_out) = table[c[:, 0]] (+ spk_table[c[:, 1, 0]]), regulated by the int64 durations ``ds`` (B, S) when
    given (t_out: the largest row total) -- pwgb_symbol_embed_forward.  Indices outside a table give NaN columns."""
    c, is64 = _index_tensor(c)
    table = _dev(table, "table")
    B, K, S = c.shape
    if spk_table is not None:
        spk_table = _dev(spk_table, "spk_table")
        if K < 2:
            raise PwgbError("symbol_embed: a speaker table needs (B, 2, S) indices")
    if ds is None:
        t_out = S
    else:
        ds = _durations(ds, B, S)
    C_ = table.shape[1]
    y = torch.empty((B, C_, int(t_out)), device=table.device, dtype=torch.float32)
    sb, sc, st = c.stride()
    prof = _Prof("symbol_embed", 0.0, 4.0 * y.numel() + c.element_size() * B * S, f"B{B} C{C_} S{S} T{t_out}")
    rc = capi.lib().pwgb_symbol_embed_forward(_p(c) if c.numel() else None, is64, sb, sc, st, _p(table), table.shape[0],
                                              _p(spk_table), spk_table.shape[0] if spk_table is not None else 0,
                                              _p(ds) if ds is not None and ds.numel() else None, B, S, C_, int(t_out),
                                              _p(y) if y.numel() else None, _stream())
    capi.check(rc, "pwgb_symbol_embed_forward")
    prof.done()
    return y


def symbol_embed_backward_raw(gy, gsym, c, ds, t_out, num_embs, num_spk=0):
    """(d_table, d_spk_table or None) of symbol_embed_raw -- pwgb_symbol_embed_backward (deterministic)."""
    c, is64 = _index_tensor(c)
    B, _, S = c.shape
    gy = _dev(gy, "gy") if gy is not None else None
    gsym = _dev(gsym, "gsym") if gsym is not None else None
    dev = (gy if gy is not None else gsym).device
    C_ = (gy if gy is not None else gsym).shape[1]
    d_emb = torch.empty((num_embs, C_), device=dev, dtype=torch.float32)
    d_spk = torch.empty((num_spk, C_), device=dev, dtype=torch.float32) if num_spk else None
    L = capi.lib()
    nbytes = L.pwgb_symbol_embed_backward_workspace(B, S, C_, num_embs)
    ws = torch.empty((nbytes + 3) // 4, device=dev, dtype=torch.float32)
    sb, sc, st = c.stride()
    rc = L.pwgb_symbol_embed_backward(_p(gy) if gy is not None and gy.numel() else None,
                                      _p(gsym) if gsym is not None and gsym.numel() else None, _p(c) if c.numel() else None, is64,
                                      sb, sc, st, _p(ds) if ds is not None and ds.numel() else None, B, S, C_, int(t_out), num_embs,
                                      _p(d_emb), num_spk, _p(d_spk), _p(ws), C.c_size_t(nbytes), _stream())
    capi.check(rc, "pwgb_symbol_embed_backward")
    return d_emb, d_spk


def symbol_embed(c, table, spk_table=None, ds=None, t_out=None, symbol_level=False):
    """Embedding (+ speaker) of the symbol indices ``c`` (B, 1 or 2, S), channel-major.  With durations ``ds`` the
    result is length-regulated to (B, C, t_out); ``symbol_level`` also returns the unregulated (B, C, S) embedding (the
    duration predictor's input).  Differentiable w.r.t. the tables through SymbolEmbedFn, whose backward takes the
    gradients of both outputs in one pass."""
    if _needs_grad(table, spk_table):
        from . import autograd as ag

        return ag.SymbolEmbedFn.apply(table, spk_table, c, ds, t_out, bool(symbol_level and ds is not None))
    y = symbol_embed_raw(c, table, spk_table, ds, t_out)
    if symbol_level and ds is not None:
        return y, symbol_embed_raw(c, table, spk_table)
    return y


def duration_round(x, offset=1.0, ds=None, zero_rule=True):
    """(ds, totals): ds = clamp(round(exp(x) - offset), min=0) as int64 (layers/duration_predictor.py:79-83), or the
    given int64 ``ds`` (B, S) with x None; totals (B,) the row sums.  ``zero_rule`` applies the length regulator's
    rule in place (layers/length_regulator.py:87-95): when the whole batch sums to zero, rows summing to zero become
    all ones.  One launch -- pwgb_duration_round."""
    if x is not None:
        x = _dev(x, "x")
        B, S = x.shape
        ds = torch.empty((B, S), device=x.device, dtype=torch.int64)
    else:
        B, S = ds.shape
        ds = _durations(ds, B, S)
    totals = torch.empty(B, device=ds.device, dtype=torch.int64)
    rc = capi.lib().pwgb_duration_round(_p(x) if x is not None and x.numel() else None, _p(ds) if ds.numel() else None,
                                        _p(totals) if B else None, B, S, float(offset), int(bool(zero_rule)), _stream())
    capi.check(rc, "pwgb_duration_round")
    return ds, totals


def regulated_length(totals):
    """The largest row total: the time length of the length-regulated tensor.  Sizing that tensor needs it on the host,
    so this is one device-to-host copy of B int64 (and a synchronisation) per forward with durations -- the reference
    synchronises at the same point (``ds.sum() == 0`` and ``repeat_interleave``, layers/length_regulator.py:87-97)."""
    return int(totals.cpu().max()) if totals.numel() else 0


def channel_layer_norm_raw(x, gamma, beta, eps, stats=False):
    """LayerNorm over the channels of (B, C, T) at every (b, t) -- pwgb_channel_layernorm_forward; with ``stats`` also
    returns the per-(b, t) mean and 1 / std."""
    x = _dev(x, "x")
    B, C_, T = x.shape
    y = torch.empty_like(x)
    mean = torch.empty((B, T), device=x.device, dtype=torch.float32) if stats else None
    rstd = torch.empty((B, T), device=x.device, dtype=torch.float32) if stats else None
    rc = capi.lib().pwgb_channel_layernorm_forward(_p(x) if x.numel() else None, _p(_dev(gamma, "gamma")), _p(_dev(beta, "beta")), B, C_, T,
                                                   float(eps), _p(y) if y.numel() else None,
                                                   _p(mean) if stats and mean.numel() else None,
                                                   _p(rstd) if stats and rstd.numel() else None, _stream())
    capi.check(rc, "pwgb_channel_layernorm_forward")
    return (y, mean, rstd) if stats else y


def channel_layer_norm(x, gamma, beta, eps):
    if _needs_grad(x, gamma, beta):
        from . import autograd as ag

        return ag.ChannelLayerNormFn.apply(x, gamma, beta, float(eps))
    return channel_layer_norm_raw(x, gamma, beta, eps)


def duration_loss_raw(x, ds, offset):
    """mean((x - log(ds + offset))^2) over all (B, S) as a 1-element tensor -- pwgb_duration_loss_forward."""
    x = _dev(x, "x")
    ds = _durations(ds, *x.shape)
    out = torch.empty(1, device=x.device, dtype=torch.float32)
    rc = capi.lib().pwgb_duration_loss_forward(_p(x), _p(ds), x.numel(), float(offset), _p(out), _stream())
    capi.check(rc, "pwgb_duration_loss_forward")
    return out


def duration_loss(x, ds, offset=1.0):
    if _needs_grad(x):
        from . import autograd as ag

        return ag.DurationLossFn.apply(x, ds, float(offset))
    return duration_loss_raw(x, ds, offset)


# ---- VQ-VAE bottleneck (models/vqvae.py, layers/vector_quantize_codebook.py): nearest-code search, gather and the
# decoder-input assembly -- pwgb_vq_forward / pwgb_vq_backward ----
def _long_tensor(t, shape, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.int64 or tuple(t.shape) != tuple(shape):
        raise PwgbError(f"{name}: expected a CUDA int64 tensor of shape {tuple(shape)}")
    return t.contiguous()


def vq_raw(z_e, codebook, *, indices=None, z_q=True, dec=True, l=None, global_table=None, g=None):
    """One pwgb_vq_forward launch -> (indices (B, T) int64, z_q (B, D, T) or None, dec (B, D + Cl + Cg, T) or None).
    ``z_e`` (B, D, T) is searched for its nearest codes (fp32, fixed-order sums, ties to the lower index, NaN first as
    torch.min); with ``indices`` given instead the search is skipped (VQVAE.decode).  ``dec`` is the decoder input:
    the gathered codes, then ``l`` (B, Cl, T), then ``global_table[g]`` broadcast over time.  An index outside the
    codebook or a ``g`` outside its table gives NaN columns."""
    codebook = _dev(codebook, "codebook")
    K, D = codebook.shape
    if z_e is not None:
        z_e = _dev(z_e, "z_e")
        if z_e.dim() != 3 or z_e.shape[1] != D:
            raise PwgbError(f"vq: z_e has shape {tuple(z_e.shape)}, the codebook {D} channels")
        B, _, T = z_e.shape
        indices = torch.empty((B, T), device=z_e.device, dtype=torch.int64)
    else:
        if not isinstance(indices, torch.Tensor) or indices.dim() != 2:
            raise PwgbError("vq: expected (B, T) indices")
        B, T = indices.shape
        indices = _long_tensor(indices, (B, T), "indices")
    dev = codebook.device
    Cl = Cg = ng = 0
    if l is not None:
        l = _dev(l, "l")
        if l.dim() != 3 or l.shape[0] != B or l.shape[2] != T:
            raise PwgbError(f"vq: local conditioning {tuple(l.shape)} does not match the codes' (B, T) = {(B, T)}")
        Cl = l.shape[1]
    if g is not None:
        if global_table is None:
            raise PwgbError("vq: global ids without a global table")
        global_table = _dev(global_table, "global_table")
        g = _long_tensor(g, (B,), "g")
        ng, Cg = global_table.shape
    if l is not None or g is not None:
        dec = True
    zq = torch.empty((B, D, T), device=dev, dtype=torch.float32) if z_q else None
    dc = torch.empty((B, D + Cl + Cg, T), device=dev, dtype=torch.float32) if dec else None
    if B * T == 0:
        return indices, zq, dc
    prof = _Prof("vq_forward", 2.0 * B * T * K * D if z_e is not None else 0.0,
                 4.0 * (B * T * D * (z_e is not None) + K * D + (zq.numel() if z_q else 0) + (dc.numel() if dec else 0)),
                 f"B{B} D{D} K{K} T{T} Cl{Cl} Cg{Cg}")
    rc = capi.lib().pwgb_vq_forward(_p(z_e), _p(codebook), K, _p(indices), _p(zq), _p(dc), _p(l) if Cl else None, Cl,
                                    _p(global_table) if g is not None else None, _p(g), ng, Cg, B, D, T, _stream())
    capi.check(rc, "pwgb_vq_forward")
    prof.done()
    return indices, zq, dc


def vq_backward_raw(gdec, dim, local_channels, g=None, num_global=0, want_gz=True):
    """(gz_e (B, D, T) or None, d_global_table (num_global, Cg) or None) from the decoder-input gradient
    (B, D + Cl + Cg, T) -- pwgb_vq_backward (deterministic)."""
    gdec = _dev(gdec, "gdec")
    B, Ct, T = gdec.shape
    Cg = Ct - dim - local_channels
    gz = torch.empty((B, dim, T), device=gdec.device, dtype=torch.float32) if want_gz else None
    dgt = torch.empty((num_global, Cg), device=gdec.device, dtype=torch.float32) if (g is not None and Cg > 0) else None
    nz = gdec.numel() > 0
    rc = capi.lib().pwgb_vq_backward(_p(gdec) if nz else None, B, dim, local_channels, Cg, T, _p(gz) if want_gz and nz else None, 0,
                                     _p(g) if dgt is not None else None, num_global, _p(dgt), _stream())
    capi.check(rc, "pwgb_vq_backward")
    return gz, dgt


def vq(z_e, codebook, *, l=None, global_table=None, g=None, z_q=True, st_codebook=False):
    """(dec, z_q, indices): the straight-through decoder input and the quantised codes of ``z_e`` (see vq_raw).  Under
    autograd ``dec`` carries the straight-through gradient to ``z_e``, to ``l`` and to ``global_table``; ``z_q`` the
    codebook gradient (``st_codebook``: ``dec``'s code channels carry it instead, functions.vector_quantize_straight_through)."""
    if _needs_grad(z_e, codebook, l, global_table):
        from . import autograd as ag

        return ag.VQFn.apply(z_e, codebook, l, global_table, g, bool(z_q), bool(st_codebook))
    indices, zq, dc = vq_raw(z_e, codebook, z_q=z_q, dec=True, l=l, global_table=global_table, g=g)
    return dc, zq, indices
