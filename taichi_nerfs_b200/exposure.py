"""Per-image exposure compensation (``--exposure_lr``, DESIGN.md §6k): one learned per-channel gain for every training
image, trained with the model.

Image i has a log2 exposure e_i in R^3 (stops) and gain g_i = 2^{e_i}; the radiance of every sample of its rays becomes
c' = g_i * c, so the composited colour is g_i * sum_k w_k c_k + T bg (the background is not scaled).  The exposures
start at zero and live in one fp32 buffer [N_img, 4] = (e_r, e_g, e_b, 0), with a gradient buffer and Adam moments of
the same layout (csrc/exposure.cu).  A gain common to all images trades against the field's colours, so after every
update the exposures are held at zero mean per channel; rendering uses e = 0, the mean exposure.  The update is Adam
with the model's betas, eps and device scalars (the same inf-skip, unscale and cosine schedule) at ``lr_ratio`` times
the model's learning rate.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops


class _ExposureApply(torch.autograd.Function):
    """rgbs [S, 3] -> 2^e[img(ray)] * rgbs over the rows of rays_a; the backward rewrites dL/dc' into dL/dc and adds
    the per-image exposure gradient into the ExposureCorrection's buffer."""

    @staticmethod
    def forward(ctx, rgbs, rays_a, img_idxs, corr):
        rgbs = rgbs.contiguous()
        out = ops.exposure_apply(rgbs, rays_a, img_idxs, corr.exposure)
        ctx.save_for_backward(out, rays_a, img_idxs)
        ctx.corr = corr
        return out

    @staticmethod
    def backward(ctx, dout):
        out, rays_a, img_idxs = ctx.saved_tensors
        d = dout.to(out.dtype).contiguous().clone()
        # no found_inf here: optimizer_step clears the flag before its update, whose finite check covers this gradient
        ops.exposure_bwd(out, d, rays_a, img_idxs, ctx.corr.exposure, ctx.corr.grad)
        return d, None, None, None


class ExposureCorrection:
    """Per-image log2 exposures of ``n_img`` training images on ``device``.  ``lr_ratio`` = exposure_lr / lr: the
    exposures' learning rate relative to the model's at every step."""

    def __init__(self, n_img: int, lr_ratio: float, device):
        if not (math.isfinite(lr_ratio) and lr_ratio >= 0):
            raise ValueError(f"ExposureCorrection: lr_ratio must be finite and >= 0, got {lr_ratio}")
        if int(n_img) <= 0:
            raise ValueError(f"ExposureCorrection: n_img must be > 0, got {n_img}")
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("ExposureCorrection: the exposures must be on a CUDA device")
        self.n_img = int(n_img)
        self.lr_ratio = float(lr_ratio)
        z = lambda: torch.zeros(self.n_img, 4, device=device, dtype=torch.float32)  # noqa: E731
        self.exposure, self.grad, self.exp_avg, self.exp_avg_sq = z(), z(), z(), z()

    def apply(self, rgbs, rays_a, img_idxs):
        """Autograd: the rows rgbs [S, 3] of the rays rays_a [n, 3] (int32) of images img_idxs [n] (or one index) under
        their images' gains."""
        idx = torch.as_tensor(img_idxs, device=rgbs.device).to(torch.int64).reshape(-1)
        return _ExposureApply.apply(rgbs, rays_a.contiguous(), idx, self)

    def enqueue_adam(self, trainer):
        """The exposures' Adam step and zero-mean projection on the trainer's device scalars (after its
        ngp_adam_hyper_update)."""
        ops.exposure_adam(self.exposure, self.grad, self.exp_avg, self.exp_avg_sq, trainer.hyper, self.lr_ratio,
                          found_inf=trainer.found_inf, beta1=trainer.betas[0], beta2=trainer.betas[1], eps=trainer.eps)

    def state(self):
        return [self.exposure, self.grad, self.exp_avg, self.exp_avg_sq]

    def exposures(self) -> np.ndarray:
        """[N_img, 3] float32 log2 exposures (stops)."""
        return self.exposure[:, :3].detach().cpu().numpy().astype(np.float32)
