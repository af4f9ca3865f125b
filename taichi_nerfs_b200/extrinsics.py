"""Camera extrinsics refinement (``--extrinsics_lr``, DESIGN.md §6i): one pose correction per training image, trained
with the model.

Image i's camera-to-world pose (R_i, o_i) becomes R'_i = Exp(omega_i) R_i (a world-frame rotation about the camera
centre, Rodrigues) and o'_i = o_i + tau_i.  The corrections start at zero and live in one fp32 buffer [N_img, 8] =
(omega[3], 0, tau[3], 0), with a gradient buffer and Adam moments of the same layout (csrc/pose.cu).  The gradient
reaches a pose through the sample positions x_s = o' + t_s d' only; the colour network's direction input is held
constant.  The update is Adam with the model's betas, eps and device scalars (the same inf-skip, unscale and cosine
schedule) at ``lr_ratio`` times the model's learning rate.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops


def so3_exp_np(w):
    """Exp of rotation vectors w [..., 3] -> [..., 3, 3], fp64 (Rodrigues, series near 0)."""
    w = np.asarray(w, np.float64)
    t2 = (w * w).sum(-1)[..., None, None]
    t = np.sqrt(t2)
    small = t2 < 1e-6
    ts = np.where(small, 1.0, t)
    A = np.where(small, 1 - t2 / 6 + t2 * t2 / 120, np.sin(ts) / ts)
    B = np.where(small, 0.5 - t2 / 24 + t2 * t2 / 720, 2 * np.sin(ts / 2) ** 2 / np.where(small, 1.0, t2))
    K = np.zeros(w.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -w[..., 2], w[..., 1], -w[..., 0]
    K[..., 1, 0], K[..., 2, 0], K[..., 2, 1] = w[..., 2], -w[..., 1], w[..., 0]
    return np.eye(3) + A * K + B * (K @ K)


class PoseRefinement:
    """Per-image pose corrections of a training set of poses [N_img, 3, 4] (camera-to-world) on one device.
    ``lr_ratio`` = extrinsics_lr / lr: the corrections' learning rate relative to the model's at every step."""

    def __init__(self, poses, lr_ratio: float):
        if not (math.isfinite(lr_ratio) and lr_ratio >= 0):
            raise ValueError(f"PoseRefinement: lr_ratio must be finite and >= 0, got {lr_ratio}")
        P = poses.detach().to(torch.float32).reshape(-1, 3, 4).contiguous()
        if not P.is_cuda:
            raise ValueError("PoseRefinement: the poses must be on a CUDA device")
        self.poses = P
        self.n_img = P.shape[0]
        self.lr_ratio = float(lr_ratio)
        z = lambda: torch.zeros(self.n_img, 8, device=P.device, dtype=torch.float32)  # noqa: E731
        self.corr, self.grad, self.exp_avg, self.exp_avg_sq = z(), z(), z(), z()

    @property
    def omega(self):
        return self.corr[:, 0:3]

    @property
    def tau(self):
        return self.corr[:, 4:7]

    def rays(self, directions, img_idxs, rays_o=None, rays_d=None):
        """(rays_o, rays_d) of camera directions [n, 3] in images img_idxs [n] (or one index) under the corrected
        poses."""
        return ops.pose_apply(directions, img_idxs, self.poses, self.corr, rays_o, rays_d)

    def accumulate(self, dx, ts, rays_a, img_idxs, rays_d, n_rays_dev=None, found_inf=None):
        """grad += the pose gradient of one batch from its sample gradients dx = dL/dx_s (csrc/pose.cu)."""
        ops.pose_grad(dx, ts, rays_a, img_idxs, rays_d, self.grad, n_rays_dev=n_rays_dev, found_inf=found_inf)

    def enqueue_adam(self, trainer):
        """The corrections' Adam step on the trainer's device scalars (after its ngp_adam_hyper_update)."""
        ops.pose_adam(self.corr, self.grad, self.exp_avg, self.exp_avg_sq, trainer.hyper, self.lr_ratio,
                      found_inf=trainer.found_inf, beta1=trainer.betas[0], beta2=trainer.betas[1], eps=trainer.eps)

    def state(self):
        return [self.corr, self.grad, self.exp_avg, self.exp_avg_sq]

    def refined_poses(self) -> np.ndarray:
        """[N_img, 3, 4] float32 corrected camera-to-world poses (fp64 Rodrigues, rounded once)."""
        c = self.corr.detach().cpu().numpy().astype(np.float64)
        P = self.poses.cpu().numpy().astype(np.float64)
        out = np.empty_like(P)
        out[:, :, :3] = so3_exp_np(c[:, 0:3]) @ P[:, :, :3]
        out[:, :, 3] = P[:, :, 3] + c[:, 4:7]
        return out.astype(np.float32)

    def mean_correction(self):
        """(mean |omega| in degrees, mean |tau|) over the images."""
        c = self.corr.detach().cpu().numpy().astype(np.float64)
        return (float(np.degrees(np.linalg.norm(c[:, 0:3], axis=1)).mean()),
                float(np.linalg.norm(c[:, 4:7], axis=1).mean()))
