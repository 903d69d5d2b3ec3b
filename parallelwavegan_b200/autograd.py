"""torch.autograd glue for the train step (bin/train.py:189-340): every Function's forward AND
backward run libpwgb kernels.  Data gradients reuse the forward kernels (dgrad of a stride-1 conv =
conv with the transposed, tap-flipped weight -> tensor-core path; dgrad of a strided conv = poly-phase
conv-transpose); weight gradients use pwgb_conv1d_wgrad.  Weight / spectral-norm
re-parametrisation stays in PyTorch on the (tiny) weight tensors, so its backward is PyTorch's."""
import ctypes as C

import torch

from . import capi, ops
from .capi import PwgbError


def _pair(p):
    return (p, p) if isinstance(p, int) else (int(p[0]), int(p[1]))


class Conv1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias, residual, stride, padding, dilation, groups, pad_mode, pre_slope, post_act, post_slope,
                out_scale, period):
        if pad_mode != "zero" and (stride != 1 or period != 1):
            raise PwgbError("training through strided / period convs with reflect or replicate padding is not supported")
        y = ops.conv1d_raw(x, w, bias, stride=stride, padding=padding, dilation=dilation, groups=groups, pad_mode=pad_mode,
                           pre_slope=pre_slope, post_act=post_act, post_slope=post_slope, residual=residual,
                           out_scale=out_scale, period=period)
        ctx.cfg = (stride, _pair(padding), dilation, groups, pre_slope, post_act, post_slope, out_scale, period)
        ctx.pad_mode = pad_mode
        ctx.has_bias = bias is not None
        ctx.has_res = residual is not None
        ctx.w3 = (w.shape[0], w.shape[1], w.shape[2])
        ctx.w_shape = tuple(w.shape)
        ctx.x_shape = tuple(x.shape)
        act_out = None
        if post_act:
            act_out = y
            if residual is not None or out_scale != 1.0:
                # the activation derivative needs act(z) = y / out_scale - residual
                act_out = torch.empty_like(y)
                ops.axpby(1.0 / out_scale, y, 0.0, act_out)
                if residual is not None:
                    ops.axpby(-1.0, residual, 1.0, act_out)
        ctx.save_for_backward(x, w, act_out)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w, y = ctx.saved_tensors
        stride, (pl, pr), dil, groups, pre_slope, post_act, post_slope, out_scale, P = ctx.cfg
        gy = gy.contiguous()
        need_x, need_w, need_b, need_r = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        g_res = None
        if ctx.has_res and need_r:
            g_res = gy if out_scale == 1.0 else ops.act_backward("scale", gy, scale=out_scale)
        if post_act == "tanh":
            gz = ops.act_backward("tanh", gy, y, scale=out_scale)
        elif post_act == "lrelu":
            gz = ops.act_backward("lrelu", gy, y, slope=post_slope, scale=out_scale)
        elif out_scale != 1.0:
            gz = ops.act_backward("scale", gy, scale=out_scale)
        else:
            gz = gy
        cout, cin_g, K = ctx.w3
        w3 = w.reshape(cout, cin_g, K)
        gb = ops.bias_grad(gz, cout) if (ctx.has_bias and need_b) else None
        gw = None
        if ctx.pad_mode != "zero" and (pl or pr):
            # reflect / replicate padding: the gradients are those of a *valid* conv over the explicitly
            # padded signal, folded back through the adjoint of the padding (stride 1, period 1 only)
            T = x.shape[2]
            if need_w:
                xp = ops.pad1d(x, pl, pr, ctx.pad_mode)
                gw = ops.conv1d_wgrad(xp, gz, ctx.w3, stride=1, padding=0, dilation=dil, groups=groups, x_slope=pre_slope).reshape(ctx.w_shape)
                del xp
            gx = None
            if need_x:
                cout_g = cout // groups
                wt = w3.detach().reshape(groups, cout_g, cin_g, K).transpose(1, 2).flip(-1).reshape(groups * cin_g, cout_g, K).contiguous()
                full = dil * (K - 1)
                gxp = ops.conv1d_raw(gz, wt, None, padding=(full, full), dilation=dil, groups=groups)
                gx = ops.pad1d_backward(gxp, T, pl, pr, ctx.pad_mode)
                if pre_slope != 1.0:
                    ops.act_backward("lrelu", gx, x, slope=pre_slope, out=gx)
            return gx, gw, gb, g_res, None, None, None, None, None, None, None, None, None, None
        if need_w:
            gw = ops.conv1d_wgrad(x, gz, ctx.w3, stride=stride, padding=pl, dilation=dil, groups=groups, x_slope=pre_slope, period=P)
            gw = gw.reshape(ctx.w_shape)
        gx = None
        if need_x:
            B, cin = x.shape[0], x.shape[1]
            L = x.numel() // (B * cin)
            t_in = (L + P - 1) // P
            t_out = gz.numel() // (B * cout * P)
            if stride == 1:
                # dgrad = conv of gz with the transposed, tap-flipped weight (layout change on the weight only)
                cout_g = cout // groups
                wt = w3.detach().reshape(groups, cout_g, cin_g, K).transpose(1, 2).flip(-1).reshape(groups * cin_g, cout_g, K).contiguous()
                pl2 = dil * (K - 1) - pl
                pr2 = t_in - t_out - pl2 + dil * (K - 1)
                gxe = ops.conv1d_raw(gz, wt, None, padding=(pl2, pr2), dilation=dil, groups=groups, period=P)
            else:
                if dil != 1 or pl != pr:
                    raise PwgbError("backward of a strided conv with dilation / asymmetric padding is not supported")
                op = t_in - ((t_out - 1) * stride - 2 * pl + K)
                if not 0 <= op < stride:
                    raise PwgbError("strided dgrad: inconsistent lengths")
                gxe = ops.conv_transpose1d_raw(gz, w3.detach(), None, stride=stride, padding=pl, output_padding=op, groups=groups, period=P)
            if pre_slope != 1.0:
                if P > 1 and t_in * P != L:
                    raise PwgbError("pre-activation on a reflect-extended period input is not supported")
                ops.act_backward("lrelu", gxe, x, slope=pre_slope, out=gxe)
            if P > 1 and t_in * P != L:
                # first MPD layer: fold the reflect extension back (hifigan.py:365-369): x_ext[T+m] = x[T-2-m]
                flat = gxe.reshape(B, cin, t_in * P)
                gx = flat[:, :, :L].contiguous()
                n_pad = t_in * P - L
                idx = torch.arange(L - 2, L - 2 - n_pad, -1, device=gx.device)
                gx[:, :, idx] += flat[:, :, L:]
                gx = gx.reshape(ctx.x_shape)
            else:
                gx = gxe.reshape(ctx.x_shape)
        return gx, gw, gb, g_res, None, None, None, None, None, None, None, None, None, None


def conv1d(x, w, bias=None, *, stride=1, padding=0, dilation=1, groups=1, pad_mode="zero", pre_slope=1.0, pre_gate=False,
           post_act=None, post_slope=0.0, residual=None, out_scale=1.0, out=None, accumulate=False, period=1):
    if pre_gate or out is not None or accumulate:
        raise PwgbError("gate / in-place accumulate variants are inference-only (no backward kernel)")
    return Conv1dFn.apply(x, w, bias, residual, stride, padding, dilation, groups, pad_mode, float(pre_slope), post_act,
                          float(post_slope), float(out_scale), int(period))


class ConvTranspose1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias, stride, padding, output_padding, pre_slope):
        y = ops.conv_transpose1d_raw(x, w, bias, stride=stride, padding=padding, output_padding=output_padding, pre_slope=pre_slope)
        ctx.cfg = (stride, padding, output_padding, pre_slope)
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, w)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        stride, padding, _, pre_slope = ctx.cfg
        gy = gy.contiguous()
        cin, cout, K = w.shape
        gb = ops.bias_grad(gy, cout) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        gw = None
        if ctx.needs_input_grad[1]:
            # dw[ci, co, k] = sum_t lrelu(x)[ci, t] * gy[co, t*s - p + k]: the conv wgrad with the roles of the
            # two operands swapped ("x" = gy, gradient operand = pre-activated x)
            gw = ops.conv1d_wgrad(gy, x, (cin, cout, K), stride=stride, padding=padding, g_slope=pre_slope)
        gx = None
        if ctx.needs_input_grad[0]:
            gx = ops.conv1d(gy, w.detach(), None, stride=stride, padding=padding)  # (cin, cout, K) read as a conv weight; strided -> space-to-depth + tensor cores
            if gx.shape[-1] != x.shape[-1]:
                raise PwgbError("conv_transpose dgrad: length mismatch")
            if pre_slope != 1.0:
                ops.act_backward("lrelu", gx, x, slope=pre_slope, out=gx)
        return gx, gw, gb, None, None, None, None


def conv_transpose1d(x, w, bias=None, *, stride, padding=0, output_padding=0, pre_slope=1.0, groups=1, period=1):
    if groups != 1 or period != 1:
        raise PwgbError("grouped / period conv_transpose is only used as a dgrad (no second-order support)")
    return ConvTranspose1dFn.apply(x, w, bias, stride, padding, output_padding, float(pre_slope))


class S2DFn(torch.autograd.Function):
    """Space-to-depth along time (strided convs on the tensor-core path); backward = the adjoint gather."""

    @staticmethod
    def forward(ctx, x, groups, stride, pad_left, rows_out, period, cgo=0):
        ctx.cfg = (tuple(x.shape), groups, stride, pad_left, period, cgo)
        return ops.s2d_raw(x, groups, stride, pad_left, rows_out, period, cgo)

    @staticmethod
    def backward(ctx, gy):
        shape, groups, stride, pad_left, period, cgo = ctx.cfg
        return ops.s2d_backward_raw(gy.contiguous(), shape, groups, stride, pad_left, period, cgo), None, None, None, None, None, None


class AvgPool1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, kernel_size, stride, padding, count_include_pad):
        ctx.cfg = (kernel_size, stride, padding, count_include_pad, x.shape)
        return ops.avg_pool1d_raw(x, kernel_size, stride, padding, count_include_pad)

    @staticmethod
    def backward(ctx, gy):
        k, s, p, inc, shape = ctx.cfg
        gy = gy.contiguous()
        gx = torch.empty(shape, device=gy.device, dtype=torch.float32)
        rc = capi.lib().pwgb_avg_pool1d_backward(ops._p(gy), ops._p(gx), shape[0] * shape[1], shape[2], int(k), int(s), int(p),
                                                 int(bool(inc)), ops._stream())
        capi.check(rc, "pwgb_avg_pool1d_backward")
        return gx, None, None, None, None


class ReduceMeanFn(torch.autograd.Function):
    """weight * mean f(x [, y]) as a 1-element tensor (GAN loss terms)."""

    @staticmethod
    def forward(ctx, x, y, mode, c, s, weight):
        ctx.cfg = (mode, c, s, weight)
        ctx.save_for_backward(x, y)
        return ops.reduce_mean_raw(mode, x, y, c, s, weight)

    @staticmethod
    def backward(ctx, gout):
        x, y = ctx.saved_tensors
        mode, c, s, weight = ctx.cfg
        gout = gout.contiguous().reshape(1)
        gx = torch.empty_like(x)
        xc = x.contiguous()
        rc = capi.lib().pwgb_reduce_mean_backward(ops._REDUCE[mode], ops._p(xc), ops._p(y.contiguous()) if y is not None else None,
                                                  x.numel(), c, s, weight, ops._p(gout), ops._p(gx), 0, ops._stream())
        capi.check(rc, "pwgb_reduce_mean_backward")
        gy = None
        if y is not None and ctx.needs_input_grad[1]:
            gy = ops.act_backward("scale", gx, scale=-1.0)
        return gx, gy, None, None, None, None


class MelLossFn(torch.autograd.Function):
    """MelSpectrogramLoss.forward (losses/mel_loss.py:150-165); gradient w.r.t. the generated signal only."""

    @staticmethod
    def forward(ctx, y_hat, y, melmat, window, fft_size, hop_size, win_length, eps, log_scale):
        ax, ay = ops.stft_amplitude(y_hat, y, fft_size, hop_size, win_length, window, eps)
        _, loss = ops.mel_project(ax, ay, melmat, eps, log_scale, want_mel=False, want_loss=True)
        ctx.cfg = (fft_size, hop_size, win_length, eps, log_scale)
        ctx.save_for_backward(y_hat, ax, ay, melmat, window)
        return loss

    @staticmethod
    def backward(ctx, gout):
        y_hat, ax, ay, melmat, window = ctx.saved_tensors
        fft_size, hop_size, win_length, eps, log_scale = ctx.cfg
        B, frames, bins = ax.shape
        L = capi.lib()
        gout = gout.contiguous().reshape(1)
        dax = torch.empty_like(ax)
        rc = L.pwgb_mel_project_backward(B, frames, bins, melmat.shape[1], ops._p(ax), ops._p(ay), ops._p(melmat), float(eps),
                                         float(log_scale), ops._p(gout), ops._p(dax), ops._stream())
        capi.check(rc, "pwgb_mel_project_backward")
        d = capi.StftDesc(batch=B, t=y_hat.shape[1], n_fft=int(fft_size), hop=int(hop_size), win_length=int(win_length), clamp_eps=float(eps))
        dx = torch.zeros_like(y_hat)
        rc = L.pwgb_stft_amplitude_backward(C.byref(d), ops._p(y_hat), ops._p(window), ops._p(ax), ops._p(dax), ops._p(dx), ops._stream())
        capi.check(rc, "pwgb_stft_amplitude_backward")
        return dx, None, None, None, None, None, None, None, None


class ScaledSumFn(torch.autograd.Function):
    """sum_i a * x_i (the MRF average cs / num_blocks of hifigan.py:187-190) -- pwgb_axpby."""

    @staticmethod
    def forward(ctx, a, *xs):
        ctx.a = a
        ctx.n = len(xs)
        out = torch.empty_like(xs[0])
        if len(xs) > 2:  # one pass over all inputs (pwgb_scaled_sum) instead of n read-modify-write passes
            xs = [x.contiguous() for x in xs]
            table = torch.tensor([x.data_ptr() for x in xs], dtype=torch.int64).to(out.device, non_blocking=True)
            aligned = all(x.data_ptr() % 16 == 0 for x in xs)
            rc = capi.lib().pwgb_scaled_sum(ops._p(table), len(xs), float(a), ops._p(out), out.numel(), int(aligned), ops._stream())
            capi.check(rc, "pwgb_scaled_sum")
            # xs / table may be released right away: the caching allocator reuses memory in stream order, after this launch
            return out
        for i, x in enumerate(xs):
            ops.axpby(a, x, 0.0 if i == 0 else 1.0, out)
        return out

    @staticmethod
    def backward(ctx, g):
        gs = ops.act_backward("scale", g.contiguous(), scale=ctx.a)
        return (None,) + (gs,) * ctx.n


# --------------------------------------------------------------------------
# Parallel WaveGAN training pieces (config C3)
# --------------------------------------------------------------------------


class GateFn(torch.autograd.Function):
    """z = tanh(g[:, :H]) * sigmoid(g[:, H:])  (layers/residual_block.py:128)."""

    @staticmethod
    def forward(ctx, g):
        g = g.contiguous()
        B, C2, T = g.shape
        z = torch.empty((B, C2 // 2, T), device=g.device, dtype=torch.float32)
        rc = capi.lib().pwgb_gate_forward(ops._p(g), ops._p(z), B, C2 // 2, T, ops._stream())
        capi.check(rc, "pwgb_gate_forward")
        ctx.save_for_backward(g)
        return z

    @staticmethod
    def backward(ctx, gz):
        (g,) = ctx.saved_tensors
        B, C2, T = g.shape
        gg = torch.empty_like(g)
        rc = capi.lib().pwgb_gate_backward(ops._p(g), ops._p(gz.contiguous()), ops._p(gg), B, C2 // 2, T, ops._stream())
        capi.check(rc, "pwgb_gate_backward")
        return gg


class UpsampleFirFn(torch.autograd.Function):
    """One stage of the conditioning upsampler (layers/upsample.py:122-128) with both adjoints."""

    @staticmethod
    def forward(ctx, x, fir, scale, out_channels):
        y = ops.upsample_fir(x, fir, scale, out_channels=out_channels)
        ctx.scale = scale
        ctx.fir_shape = tuple(fir.shape)
        ctx.save_for_backward(x, fir)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, fir = ctx.saved_tensors
        B, Cc, T = x.shape
        gy = gy.contiguous()
        oc = gy.shape[1]
        need_x, need_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gx = torch.empty_like(x) if need_x else None
        df = torch.empty(2 * ctx.scale + 1, device=x.device, dtype=torch.float32) if need_f else None
        f1 = fir.detach().reshape(-1).contiguous()
        rc = capi.lib().pwgb_upsample_fir_backward(B * Cc, Cc, T, int(ctx.scale), ops._p(x), ops._p(f1), ops._p(gy),
                                                   oc * T * ctx.scale, ops._p(gx), ops._p(df), ops._stream())
        capi.check(rc, "pwgb_upsample_fir_backward")
        return gx, (df.reshape(ctx.fir_shape) if need_f else None), None, None


class MrStftLossFn(torch.autograd.Function):
    """MultiResolutionSTFTLoss.forward (losses/stft_loss.py:146-170) on materialised magnitudes, with the
    gradient w.r.t. the predicted signal x.  Returns a 2-element tensor [sc, mag]."""

    @staticmethod
    def forward(ctx, x, y, fft_sizes, hop_sizes, win_lengths, *windows):
        L = capi.lib()
        n_res = len(fft_sizes)
        out = torch.zeros(2, device=x.device, dtype=torch.float32)
        saved = []
        ws = torch.empty(3 * 1024, device=x.device, dtype=torch.float64)
        for i, (f, h, wl, win) in enumerate(zip(fft_sizes, hop_sizes, win_lengths, windows)):
            ax, ay = ops.stft_amplitude(x, y, f, h, wl, win, 1e-7)
            sums = torch.empty(3, device=x.device, dtype=torch.float64)
            rc = L.pwgb_stft_loss_terms(ops._p(ax), ops._p(ay), ax.numel(), 1.0 / n_res, int(i > 0), ops._p(out), ops._p(sums),
                                        ops._p(ws), 3 * 1024, ops._stream())
            capi.check(rc, "pwgb_stft_loss_terms")
            saved += [ax, ay, sums]
        ctx.cfg = (tuple(fft_sizes), tuple(hop_sizes), tuple(win_lengths))
        ctx.save_for_backward(x, *windows, *saved)
        return out

    @staticmethod
    def backward(ctx, gout):
        fft_sizes, hop_sizes, win_lengths = ctx.cfg
        n_res = len(fft_sizes)
        t = ctx.saved_tensors
        x, windows, saved = t[0], t[1 : 1 + n_res], t[1 + n_res :]
        gout = gout.contiguous()
        L = capi.lib()
        dx = torch.zeros_like(x)
        for i in range(n_res):
            ax, ay, sums = saved[3 * i : 3 * i + 3]
            dax = torch.empty_like(ax)
            rc = L.pwgb_stft_loss_dmag(ops._p(ax), ops._p(ay), ax.numel(), ops._p(sums), ops._p(gout), 1.0 / n_res, ops._p(dax), ops._stream())
            capi.check(rc, "pwgb_stft_loss_dmag")
            d = capi.StftDesc(batch=x.shape[0], t=x.shape[1], n_fft=int(fft_sizes[i]), hop=int(hop_sizes[i]),
                              win_length=int(win_lengths[i]), clamp_eps=1e-7)
            rc = L.pwgb_stft_amplitude_backward(C.byref(d), ops._p(x), ops._p(windows[i]), ops._p(ax), ops._p(dax), ops._p(dx), ops._stream())
            capi.check(rc, "pwgb_stft_amplitude_backward")
        return (dx, None, None, None, None) + (None,) * n_res


# ---------------------------------------------------------------------------------------------------------------
# StyleMelGAN generator glue (layers/tade_res_block.py:52-160 under autograd)
# ---------------------------------------------------------------------------------------------------------------
class InstanceNormFn(torch.autograd.Function):
    """InstanceNorm1d (no affine) of LeakyReLU_{pre_slope}(x); the backward recomputes the row statistics from x."""

    @staticmethod
    def forward(ctx, x, eps, pre_slope):
        x = x.contiguous()
        B, Cc, T = x.shape
        y = torch.empty_like(x)
        rc = capi.lib().pwgb_instance_norm_forward(ops._p(x), ops._p(y), B * Cc, T, float(eps), float(pre_slope), ops._stream())
        capi.check(rc, "pwgb_instance_norm_forward")
        ctx.save_for_backward(x)
        ctx.eps, ctx.pre_slope = float(eps), float(pre_slope)
        return y

    @staticmethod
    def backward(ctx, gy):
        (x,) = ctx.saved_tensors
        B, Cc, T = x.shape
        gx = torch.empty_like(x)
        rc = capi.lib().pwgb_instance_norm_backward(ops._p(x), ops._p(gy.contiguous()), ops._p(gx), B * Cc, T, ctx.eps, ctx.pre_slope,
                                                    ops._stream())
        capi.check(rc, "pwgb_instance_norm_backward")
        return gx, None, None


def _nearest_backward(gy, scale):
    B, Cc, To = gy.shape
    gx = torch.empty((B, Cc, To // scale), device=gy.device, dtype=torch.float32)
    rc = capi.lib().pwgb_upsample_nearest_backward(ops._p(gy.contiguous()), ops._p(gx), B * Cc, To // scale, int(scale), ops._stream())
    capi.check(rc, "pwgb_upsample_nearest_backward")
    return gx


class UpsampleNearestFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        x = x.contiguous()
        B, Cc, T = x.shape
        y = torch.empty((B, Cc, T * scale), device=x.device, dtype=torch.float32)
        rc = capi.lib().pwgb_upsample_nearest_forward(ops._p(x), ops._p(y), B * Cc, T, int(scale), ops._stream())
        capi.check(rc, "pwgb_upsample_nearest_forward")
        ctx.scale = int(scale)
        return y

    @staticmethod
    def backward(ctx, gy):
        return _nearest_backward(gy, ctx.scale), None


class LeakyReluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, slope):
        x = x.contiguous()
        y = torch.empty_like(x)
        rc = capi.lib().pwgb_leaky_relu_forward(ops._p(x), ops._p(y), x.numel(), float(slope), ops._stream())
        capi.check(rc, "pwgb_leaky_relu_forward")
        ctx.save_for_backward(y)  # the mask can be read from the output (slope > 0 keeps the sign)
        ctx.slope = float(slope)
        return y

    @staticmethod
    def backward(ctx, gy):
        (y,) = ctx.saved_tensors
        return ops.act_backward("lrelu", gy.contiguous(), y, slope=ctx.slope), None


class TadeCombineFn(torch.autograd.Function):
    """y = cg[:, :C] * nearest(xn, scale) + cg[:, C:]  (tade_res_block.py:72-74)."""

    @staticmethod
    def forward(ctx, cg, xn, scale):
        cg, xn = cg.contiguous(), xn.contiguous()
        B, C2, T = cg.shape
        y = torch.empty((B, C2 // 2, T), device=cg.device, dtype=torch.float32)
        rc = capi.lib().pwgb_tade_combine_forward(ops._p(cg), ops._p(xn), ops._p(y), B, C2 // 2, T, int(scale), ops._stream())
        capi.check(rc, "pwgb_tade_combine_forward")
        ctx.save_for_backward(cg, xn)
        ctx.scale = int(scale)
        return y

    @staticmethod
    def backward(ctx, gy):
        cg, xn = ctx.saved_tensors
        B, C2, T = cg.shape
        gcg, gxn = torch.empty_like(cg), torch.empty_like(xn)
        rc = capi.lib().pwgb_tade_combine_backward(ops._p(cg), ops._p(xn), ops._p(gy.contiguous()), ops._p(gcg), ops._p(gxn), B, C2 // 2, T,
                                                   ctx.scale, ops._stream())
        capi.check(rc, "pwgb_tade_combine_backward")
        return gcg, gxn, None


class TadeGateFn(torch.autograd.Function):
    """y = gate(x[:, :C]) * tanh(x[:, C:]) [+ nearest(residual, scale)]  (tade_res_block.py:150-159)."""

    @staticmethod
    def forward(ctx, x, residual, scale, softmax):
        x = x.contiguous()
        residual = residual.contiguous() if residual is not None else None
        B, C2, T = x.shape
        y = torch.empty((B, C2 // 2, T), device=x.device, dtype=torch.float32)
        rc = capi.lib().pwgb_tade_gate_forward(ops._p(x), ops._p(residual), ops._p(y), B, C2 // 2, T, int(scale), int(softmax), ops._stream())
        capi.check(rc, "pwgb_tade_gate_forward")
        ctx.save_for_backward(x)
        ctx.scale, ctx.softmax, ctx.has_res = int(scale), int(softmax), residual is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        (x,) = ctx.saved_tensors
        B, C2, T = x.shape
        gy = gy.contiguous()
        gx = torch.empty_like(x)
        rc = capi.lib().pwgb_tade_gate_backward(ops._p(x), ops._p(gy), ops._p(gx), B, C2 // 2, T, ctx.softmax, ops._stream())
        capi.check(rc, "pwgb_tade_gate_backward")
        gres = _nearest_backward(gy, ctx.scale) if ctx.has_res and ctx.needs_input_grad[1] else None
        return gx, gres, None, None
