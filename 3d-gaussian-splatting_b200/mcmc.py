"""MCMC densification schedule (3DGS-MCMC, Kheradmand et al. 2024; the defaults are gsplat's `MCMCStrategy`).

An opt-in alternative to prune / clone / split: the Gaussian count grows to a hard cap `cap_max` and never beyond it,
and dead Gaussians are moved onto live ones instead of being pruned and regrown.  Per training step:

    loss.backward()                     # (and the data-parallel gradient exchange)
    mcmc.after_backward(it)             # regulariser gradients, in place on the gradient bucket
    optimizer.step()
    mcmc.after_step(it, lr_pos)         # refine steps: relocate, then grow; every step: position noise

The work is `Splatter.mcmc_relocate`, `mcmc_add`, `mcmc_noise` and `add_mcmc_regularizer_grads`; every random draw
comes from torch's generators, so data-parallel replicas seeded alike stay identical and checkpoints resume exactly.
"""
from __future__ import annotations


class MCMC:
    def __init__(self, splatter, optimizer, cap_max, refine_start=500, refine_stop=25000, refine_every=100,
                 min_opacity=0.005, noise_lr=5e5, opacity_reg=0.01, scale_reg=0.01, growth=1.05):
        if not 0 < min_opacity < 1:
            raise ValueError(f"min_opacity must be in (0, 1), not {min_opacity!r}")
        if refine_every < 1:
            raise ValueError(f"refine_every must be >= 1, not {refine_every!r}")
        self.splatter, self.optimizer = splatter, optimizer
        self.cap_max, self.growth = int(cap_max), float(growth)
        self.refine_start, self.refine_stop, self.refine_every = int(refine_start), int(refine_stop), int(refine_every)
        self.min_opacity, self.noise_lr = float(min_opacity), float(noise_lr)
        self.opacity_reg, self.scale_reg = float(opacity_reg), float(scale_reg)

    def is_refine_step(self, it):
        return self.refine_start <= it < self.refine_stop and it % self.refine_every == 0

    def after_backward(self, it):
        """The regularisers' gradients, added in place to opa.grad and scale.grad."""
        self.splatter.add_mcmc_regularizer_grads(self.opacity_reg, self.scale_reg)

    def after_step(self, it, lr_pos):
        """On refine steps relocate the dead Gaussians, then grow towards `cap_max`; then the position noise with
        scaler = lr_pos * noise_lr.  Returns dict(relocated=<CUDA int32 [1]> or None, added=<int>)."""
        out = dict(relocated=None, added=0)
        if self.is_refine_step(it):
            out["relocated"] = self.splatter.mcmc_relocate(self.optimizer, self.min_opacity)
            out["added"] = self.splatter.mcmc_add(self.cap_max, self.growth, self.optimizer,
                                                  min_opacity=self.min_opacity)
        self.splatter.mcmc_noise(float(lr_pos) * self.noise_lr)
        return out
