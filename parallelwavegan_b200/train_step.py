"""One GAN train step -- ``Trainer._train_step`` (bin/train.py:189-340) re-hosted on the libpwgb forward /
backward kernels, for every recipe family on the hot path: Parallel WaveGAN (x = (z, c), MR-STFT loss, RAdam +
gradient clipping), MelGAN / multi-band MelGAN (PQMF synthesis, sub-band STFT loss, feature matching) and
HiFi-GAN (mel loss, feature matching, Adam).  The loss wiring follows the reference line by line; the D weight
gradients of the generator phase, which the reference computes and then discards (``optimizer["discriminator"]
.zero_grad()`` at train.py:327), are not computed.

Data parallelism = one process per GPU with ``torch.nn.parallel.DistributedDataParallel`` (bucketed NCCL
gradient all-reduce overlapped with the backward), replacing the reference's apex DDP (train.py:1494-1503).
With the fused optimizers of ``parallelwavegan_b200.optimizers`` the clip + update of a whole model is three
launches right after the all-reduce."""
import torch

from .optimizers import _FusedBase


class GanTrainStep:
    def __init__(self, generator, discriminator, criterion, opt_g, opt_d, lambda_aux=45.0, lambda_adv=1.0,
                 lambda_feat_match=2.0, grad_norm_g=-1, grad_norm_d=-1, generator_train_start_steps=0,
                 discriminator_train_start_steps=0, update_prediction_after_generator_update=True, sched_g=None, sched_d=None, steps=0):
        """criterion: dict with any of ``stft`` (MultiResolutionSTFTLoss), ``sub_stft``, ``mel``, ``pqmf``, and
        ``gen_adv`` / ``dis_adv`` / ``feat_match`` and ``duration`` (DurationPredictorLoss) -- the keys of
        ``Trainer.criterion`` (train.py:1384-1451); a key that is present is used (the reference's ``use_*_loss``
        switches).  With ``duration`` the generator is a duration model called as ``G(x, ds)`` (train.py:208-213)."""
        self.g, self.d = generator, discriminator
        self.crit = criterion
        self.opt_g, self.opt_d = opt_g, opt_d
        self.sched_g, self.sched_d = sched_g, sched_d
        self.lambda_aux, self.lambda_adv, self.lambda_fm = lambda_aux, lambda_adv, lambda_feat_match
        self.grad_norm_g, self.grad_norm_d = grad_norm_g, grad_norm_d
        self.g_start, self.d_start = generator_train_start_steps, discriminator_train_start_steps
        self.update_prediction = update_prediction_after_generator_update
        self.steps = steps  # Trainer.steps: a phase runs when steps > its *_train_start_steps (so never on the very first call from 0)

    @staticmethod
    def _params(m):
        return (m.module if hasattr(m, "module") else m).parameters()

    def _update(self, opt, model, max_norm, sched):
        if isinstance(opt, _FusedBase):
            opt.step(max_grad_norm=max_norm if max_norm > 0 else None)  # clip + update: 3 launches for the whole model
        else:
            if max_norm > 0:
                torch.nn.utils.clip_grad_norm_(self._params(model), max_norm)
            opt.step()
        if sched is not None:
            sched.step()

    def _generate(self, x, ds=None):
        ds_ = None
        if "duration" in self.crit:
            y_, ds_ = self.g(x, ds)  # train.py:208-213
        else:
            y_ = self.g(*x) if isinstance(x, (tuple, list)) else self.g(x)
        y_mb_ = None
        if "pqmf" in self.crit and y_.shape[1] > 1:  # multi-band: reconstruct the full-band signal (train.py:225-227)
            y_mb_ = y_
            y_ = self.crit["pqmf"].synthesis(y_mb_)
        return y_, y_mb_, ds_

    def __call__(self, x, y, ds=None):
        """x: conditioning (B, mels, frames), the tuple (z, c) of the Parallel WaveGAN recipes, or the (B, C, S) symbol
        codes of the duration recipes with their run lengths ``ds`` (B, S); y: (B, 1, T).
        Returns a dict of loss tensors (device scalars; nothing is synchronised with the host)."""
        stats = {}
        adv_on = self.steps > self.d_start
        y_ = None
        # ---------------- generator phase (train.py:200-295)
        if self.steps > self.g_start:
            y_, y_mb_, ds_ = self._generate(x, ds)
            gen_loss = 0.0
            if ds_ is not None:
                # gen_loss starts from the duration loss, so lambda_aux (and the sub-band 0.5) scale it too (train.py:213-262)
                dur = self.crit["duration"](ds_, ds)
                stats["duration_loss"] = dur.detach()
                gen_loss = gen_loss + dur
            if "stft" in self.crit:
                sc, mag = self.crit["stft"](y_, y)
                stats["spectral_convergence_loss"], stats["log_stft_magnitude_loss"] = sc.detach(), mag.detach()
                gen_loss = gen_loss + sc + mag
            if "sub_stft" in self.crit:
                gen_loss = gen_loss * 0.5  # train.py:243
                y_mb = self.crit["pqmf"].analysis(y)
                ssc, smag = self.crit["sub_stft"](y_mb_, y_mb)
                stats["sub_spectral_convergence_loss"], stats["sub_log_stft_magnitude_loss"] = ssc.detach(), smag.detach()
                gen_loss = gen_loss + 0.5 * (ssc + smag)
            if "mel" in self.crit:
                mel = self.crit["mel"](y_, y)
                stats["mel_loss"] = mel.detach()
                gen_loss = gen_loss + mel
            gen_loss = gen_loss * self.lambda_aux  # train.py:262
            if adv_on:
                for p in self._params(self.d):
                    p.requires_grad_(False)
                p_ = self.d(y_)
                adv = self.crit["gen_adv"](p_)
                stats["adversarial_loss"] = adv.detach()
                if "feat_match" in self.crit:
                    with torch.no_grad():
                        p = self.d(y)
                    fm = self.crit["feat_match"](p_, p)
                    stats["feature_matching_loss"] = fm.detach()
                    adv = adv + self.lambda_fm * fm  # train.py:279
                gen_loss = gen_loss + self.lambda_adv * adv
            stats["generator_loss"] = gen_loss.detach()
            self.opt_g.zero_grad(set_to_none=True)
            gen_loss.backward()
            self._update(self.opt_g, self.g, self.grad_norm_g, self.sched_g)
            if adv_on:
                for p in self._params(self.d):
                    p.requires_grad_(True)
        # ---------------- discriminator phase (train.py:300-335)
        if adv_on:
            if self.update_prediction or y_ is None:
                with torch.no_grad():
                    y_, _, _ = self._generate(x, ds)
            p = self.d(y)
            p_ = self.d(y_.detach())
            real, fake = self.crit["dis_adv"](p_, p)
            dis_loss = real + fake
            stats["real_loss"], stats["fake_loss"], stats["discriminator_loss"] = real.detach(), fake.detach(), dis_loss.detach()
            self.opt_d.zero_grad(set_to_none=True)
            dis_loss.backward()
            self._update(self.opt_d, self.d, self.grad_norm_d, self.sched_d)
        self.steps += 1  # train.py:338
        return stats
