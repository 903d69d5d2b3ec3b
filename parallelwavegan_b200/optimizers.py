"""Fused multi-tensor optimizers (mirror of ``parallel_wavegan.optimizers`` + ``torch.optim.Adam`` as the
recipes use them) with global-norm gradient clipping folded into the same pass (SURVEY.md 8f-1).

``FusedAdam``  -- ``torch.optim.Adam`` semantics (amsgrad=False), the HiFi-GAN / MelGAN recipes
                  (egs/ljspeech/voc1/conf/hifigan.v1.yaml:136-163).
``RAdam``      -- the reference's own rectified Adam (optimizers/radam.py:27-99), the Parallel WaveGAN
                  recipes (conf/parallel_wavegan.v1.yaml:91-108); ``FusedRAdam`` is an alias.

Per-parameter state keeps the reference layout (``step``, ``exp_avg``, ``exp_avg_sq``), so ``state_dict()``
round-trips with the reference optimizers.  One ``step()`` is three kernel launches for the whole model
(``pwgb_mt_clip_coef`` + ``pwgb_mt_adam_step``) instead of several per parameter; it is meant to run right
after the DDP gradient all-reduce.  No CPU path: parameters must live on a CUDA device.
"""
import ctypes as C
import math

import torch

from . import capi, ops
from .capi import PwgbError

CHUNK = 8192  # elements per CTA of the multi-tensor kernels


def _bump_versions(tensors):
    setter = getattr(torch._C._autograd, "_unsafe_set_version_counter", None)
    if setter is not None:
        try:
            setter(tuple(tensors), tuple(t._version + 1 for t in tensors))
            return
        except Exception:
            pass
    with torch.no_grad():
        for t in tensors:  # in-place op on an empty view: bumps the shared version counter, launches nothing
            t.view(-1)[:0].zero_()


class _FusedBase(torch.optim.Optimizer):
    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._tables = {}
        self.last_grad_norm = None  # device tensor [total_norm, clip_coef] of the last clipped step

    # ---- device-side tables -------------------------------------------------
    def _table(self, plist):
        """(tensor table, chunk table, n_chunks, partial workspace, out2) for a list of parameters with gradients."""
        dev = plist[0].device
        rows = []
        chunks = []
        for ti, p in enumerate(plist):
            st = self.state[p]
            g = p.grad
            if g.dtype != torch.float32 or p.dtype != torch.float32 or not p.is_cuda:
                raise PwgbError("fused optimizer: parameters and gradients must be float32 CUDA tensors (no CPU fallback)")
            if not g.is_contiguous() or not p.is_contiguous():
                raise PwgbError("fused optimizer: non-contiguous parameter / gradient")
            n = p.numel()
            rows.append((p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), n))
            for c in range((n + CHUNK - 1) // CHUNK):
                chunks.append((ti, c))
        key = tuple(rows)
        ids = tuple(id(p) for p in plist)
        ent = self._tables.get(ids)
        if ent is None or ent[0] != key:  # first use, or an address changed (gradients re-allocated by zero_grad(set_to_none=True))
            t_host = torch.tensor(rows, dtype=torch.int64).pin_memory()
            c_host = torch.tensor(chunks, dtype=torch.int32).reshape(-1, 2).pin_memory()
            if ent is None and len(self._tables) >= 8:
                self._tables.clear()
            ent = (key, t_host.to(dev, non_blocking=True), c_host.to(dev, non_blocking=True), len(chunks),
                   torch.empty(max(len(chunks), 1), device=dev, dtype=torch.float32), torch.empty(2, device=dev, dtype=torch.float32),
                   (t_host, c_host))  # the pinned staging tensors stay alive until the async copies have run
            self._tables[ids] = ent
        return ent[1], ent[2], ent[3], ent[4], ent[5]

    def _init_state(self, p):
        raise NotImplementedError

    @torch.no_grad()
    def step(self, closure=None, max_grad_norm=None, write_clipped_grad=False):
        """One optimizer step.  ``max_grad_norm`` > 0 folds ``clip_grad_norm_(all parameters, max_grad_norm)``
        (global norm over every parameter of every group, like the call on ``model.parameters()`` in
        bin/train.py:289-293) into the update; the norm / coefficient stay on the device in
        ``self.last_grad_norm``.  Gradients are scaled on the fly; ``write_clipped_grad`` also writes them back."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        allp = [p for g in self.param_groups for p in g["params"] if p.grad is not None]
        if not allp:
            return loss
        for p in allp:
            if len(self.state[p]) == 0:
                self._init_state(p)
        L = capi.lib()
        stream = ops._stream()
        coef = None
        if max_grad_norm is not None and max_grad_norm > 0:
            table, chunks, nch, partial, out2 = self._table(allp)
            rc = L.pwgb_mt_clip_coef(C.c_void_p(table.data_ptr()), C.c_void_p(chunks.data_ptr()), nch, CHUNK, float(max_grad_norm),
                                     C.c_void_p(partial.data_ptr()), C.c_void_p(out2.data_ptr()), stream)
            capi.check(rc, "pwgb_mt_clip_coef")
            coef = out2
            self.last_grad_norm = out2
        for group in self.param_groups:
            gp = [p for p in group["params"] if p.grad is not None]
            # parameters of one group normally share their step count; bucket by it to stay exact otherwise
            buckets = {}
            for p in gp:
                buckets.setdefault(int(self.state[p]["step"]), []).append(p)
            for step_no, plist in buckets.items():
                table, chunks, nch, _, _ = self._table(plist)
                self._launch(L, group, table, chunks, nch, step_no + 1, coef, write_clipped_grad, stream)
                for p in plist:
                    self._bump(p)
        # the kernels wrote the parameters through raw pointers: advance autograd's version counters like an
        # in-place torch op would, so that everything keyed on them (packed weight caches, saved-tensor checks) sees the update
        _bump_versions(allp)
        return loss

    def _bump(self, p):
        self.state[p]["step"] += 1


class FusedAdam(_FusedBase):
    """``torch.optim.Adam(params, lr, betas, eps, weight_decay)`` (amsgrad=False) as one multi-tensor launch."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False):
        if amsgrad:
            raise PwgbError("FusedAdam: amsgrad has no sm_90a kernel")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False))

    def _init_state(self, p):
        st = self.state[p]
        st["step"] = torch.tensor(0.0, dtype=torch.float32)  # torch.optim.Adam keeps a (host) tensor
        st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)

    def _launch(self, L, group, table, chunks, nch, t, coef, write_grad, stream):
        b1, b2 = group["betas"]
        c1 = group["lr"] / (1.0 - b1**t)
        c2 = 1.0 / math.sqrt(1.0 - b2**t)
        rc = L.pwgb_mt_adam_step(C.c_void_p(table.data_ptr()), C.c_void_p(chunks.data_ptr()), nch, CHUNK, 0, float(group["lr"]), float(b1),
                                 float(b2), float(group["eps"]), float(group["weight_decay"]), float(c1), float(c2),
                                 C.c_void_p(coef.data_ptr()) if coef is not None else None, int(write_grad), stream)
        capi.check(rc, "pwgb_mt_adam_step")


class RAdam(_FusedBase):
    """The reference's RAdam (optimizers/radam.py:27-99): same update, same state layout, one launch."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def _init_state(self, p):
        st = self.state[p]
        st["step"] = 0
        st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)

    def _launch(self, L, group, table, chunks, nch, t, coef, write_grad, stream):
        b1, b2 = group["betas"]
        beta2_t = b2**t
        n_sma_max = 2.0 / (1.0 - b2) - 1.0
        n_sma = n_sma_max - 2.0 * t * beta2_t / (1.0 - beta2_t)
        if n_sma >= 5:  # radam.py:66-79
            step_size = math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_sma_max - 4) * (n_sma - 2) / n_sma * n_sma_max / (n_sma_max - 2)) / (1 - b1**t)
            mode = 1
        else:
            step_size = 1.0 / (1 - b1**t)
            mode = 2
        rc = L.pwgb_mt_adam_step(C.c_void_p(table.data_ptr()), C.c_void_p(chunks.data_ptr()), nch, CHUNK, mode, float(group["lr"]), float(b1),
                                 float(b2), float(group["eps"]), float(group["weight_decay"]), float(step_size * group["lr"]), 1.0,
                                 C.c_void_p(coef.data_ptr()) if coef is not None else None, int(write_grad), stream)
        capi.check(rc, "pwgb_mt_adam_step")


FusedRAdam = RAdam
