"""Mirror of ``parallel_wavegan.functions`` (functions/vector_quantizer.py): vector quantisation of (B, *, D) inputs
against a (K, D) codebook on the VQ kernel (pwgb_vq_forward).  The kernel reads channel-major (B, D, T) codes, so a
(B, T, D) input that is the transposed view of a channel-major tensor (what VQCodebook passes) is read in place;
any other layout is copied to it first."""
import torch

from . import ops
from .capi import PwgbError


def _channel_major(inputs, codebook):
    if not isinstance(inputs, torch.Tensor) or inputs.dim() < 2 or inputs.shape[-1] != codebook.shape[1]:
        raise PwgbError(f"vector_quantize: inputs of shape {tuple(getattr(inputs, 'shape', ()))} do not end in embed_dim "
                        f"{codebook.shape[1]}")
    x = inputs if inputs.dim() == 3 else inputs.reshape(1, -1, inputs.shape[-1])
    return x.transpose(1, 2)  # (B, D, T): a contiguous tensor when inputs is the transposed view of one


class VectorQuantization(torch.autograd.Function):
    """functions/vector_quantizer.py:16-63: nearest-code indices (B, *); not differentiable."""

    @staticmethod
    def forward(ctx, inputs, codebook):
        indices, _, _ = ops.vq_raw(_channel_major(inputs, codebook).detach(), codebook.detach(), z_q=False, dec=False)
        indices = indices.reshape(inputs.shape[:-1])
        ctx.mark_non_differentiable(indices)
        return indices

    @staticmethod
    def backward(ctx, grad_output):
        raise RuntimeError(
            "Trying to call `.grad()` on graph containing "
            "`VectorQuantization`. The function `VectorQuantization` "
            "is not differentiable. Use `VectorQuantizationStraightThrough` "
            "if you want a straight-through estimator of the gradient."
        )


def vector_quantize(inputs, codebook):
    return VectorQuantization.apply(inputs, codebook)


def vector_quantize_straight_through(inputs, codebook):
    """functions/vector_quantizer.py:66-120 -> (codes (B, *, D), flattened indices): the codes' gradient is passed
    straight through to ``inputs`` and index-added into ``codebook``."""
    codes, _, indices = ops.vq(_channel_major(inputs, codebook), codebook, z_q=False, st_codebook=True)
    return codes.transpose(1, 2).reshape(inputs.shape), indices.reshape(-1)
