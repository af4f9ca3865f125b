"""Camera intrinsics (DESIGN.md §6l): the lens-distortion camera of the disk loaders (``--lens_distortion``) and a
learned focal length and principal point (``--intrinsics_lr``).

A ``Camera`` is a model and its parameters in pixels: (fx, fy, cx, cy) scaled to the loaded image size, and the
distortion terms (k1, k2, p1, p2), unscaled because they act on normalised coordinates.  Pixel directions are
(x_u, y_u, 1) with (x_u, y_u) the undistorted coordinates of the pixel's distorted ones (csrc/camera.cu).

``IntrinsicsRefinement`` trains one correction (a, b_x, b_y) for the training set's camera: fx' = fx e^a, fy' = fy e^a
(one log focal scale keeps the calibrated aspect ratio), cx' = cx + W b_x, cy' = cy + H b_y.  The distortion terms
stay as calibrated.  The gradient reaches the corrections through the sample positions x_s = o + t_s R' c only (the
colour network's direction input and each sample's t are held constant, as in §6i).  Every ray's gradient goes to its
own row of a per-ray buffer, and the Adam kernel reduces the rows in ray order, so the update is bitwise reproducible.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import torch

from . import ops

# model name -> (id of include/ngp_b200.h, number of distortion terms it has)
MODELS = {'PINHOLE': (0, 0), 'SIMPLE_PINHOLE': (0, 0), 'SIMPLE_RADIAL': (1, 1), 'RADIAL': (2, 2), 'OPENCV': (3, 4)}


@dataclasses.dataclass(frozen=True)
class Camera:
    """One pinhole-plus-distortion camera: ``model`` is a key of MODELS, ``dist`` = (k1, k2, p1, p2)."""
    model: str
    fx: float
    fy: float
    cx: float
    cy: float
    dist: tuple = (0.0, 0.0, 0.0, 0.0)

    def __post_init__(self):
        if self.model not in MODELS:
            raise ValueError(f"camera model {self.model} is not supported ({', '.join(MODELS)} are)")
        d = tuple(float(v) for v in self.dist)
        if len(d) != 4 or any(d[MODELS[self.model][1]:]):
            raise ValueError(f"{self.model}: distortion terms {self.dist} must be (k1, k2, p1, p2) with only the "
                             f"model's first {MODELS[self.model][1]} non-zero")
        object.__setattr__(self, 'dist', d)
        vals = (self.fx, self.fy, self.cx, self.cy) + d
        if not all(math.isfinite(v) for v in vals) or not (self.fx > 0 and self.fy > 0):
            raise ValueError(f"camera parameters must be finite with focal lengths > 0, got {vals}")

    @property
    def model_id(self) -> int:
        return MODELS[self.model][0]

    @property
    def params(self):
        return (float(self.fx), float(self.fy), float(self.cx), float(self.cy)) + self.dist

    @property
    def has_distortion(self) -> bool:
        return any(self.dist)

    def K(self):
        """The 3 x 3 fp32 intrinsics matrix the loaders keep (each entry rounded once)."""
        return torch.tensor([[self.fx, 0, self.cx], [0, self.fy, self.cy], [0, 0, 1]], dtype=torch.float32)

    def as_dict(self):
        k1, k2, p1, p2 = self.dist
        return dict(model=self.model, fx=self.fx, fy=self.fy, cx=self.cx, cy=self.cy, k1=k1, k2=k2, p1=p1, p2=p2)


def distort_np(camera: Camera, x, y):
    """The distortion map D of ``camera`` on undistorted normalised coordinates (numpy or torch, any dtype)."""
    k1, k2, p1, p2 = camera.dist
    r2 = x * x + y * y
    rad = 1.0 + k1 * r2 + k2 * r2 * r2
    return (x * rad + 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x),
            y * rad + p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y)


def border_pixels(W: int, H: int):
    """int64 indices of the pixels on the border of a W x H image."""
    u, v = np.arange(W), np.arange(H)
    p = np.concatenate([u, (H - 1) * W + u, v * W, v * W + W - 1])
    return np.unique(p).astype(np.int64)


def unproject_table(camera: Camera, W: int, H: int, device):
    """Directions [W*H, 3] fp32 of every pixel; raises if any pixel is not invertible (beyond the fold of D)."""
    n_bad = torch.zeros(1, device=device, dtype=torch.int32)
    dirs = ops.camera_unproject(camera, W, H, n_bad=n_bad, device=device)
    bad = int(n_bad.item())
    if bad:
        raise ValueError(f"{camera.model} camera {camera.dist}: {bad} of {W * H} pixels are not invertible (beyond "
                         f"the fold of the distortion polynomial)")
    return dirs


class IntrinsicsRefinement:
    """The training camera's intrinsics corrections on one device.  ``poses`` [N_img, 3, 4] are the training poses
    (the rays' rotations, which the gradient is chained through); ``lr_ratio`` = intrinsics_lr / lr."""

    def __init__(self, camera: Camera, W: int, H: int, lr_ratio: float, poses):
        if not (math.isfinite(lr_ratio) and lr_ratio >= 0):
            raise ValueError(f"IntrinsicsRefinement: lr_ratio must be finite and >= 0, got {lr_ratio}")
        P = poses.detach().to(torch.float32).reshape(-1, 3, 4).contiguous()
        if not P.is_cuda:
            raise ValueError("IntrinsicsRefinement: the poses must be on a CUDA device")
        self.camera, self.W, self.H, self.lr_ratio, self.poses = camera, int(W), int(H), float(lr_ratio), P
        self.n_img = P.shape[0]
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, device=P.device, dtype=dtype)  # noqa: E731
        self.corr, self.exp_avg, self.exp_avg_sq = z(1, 4), z(1, 4), z(1, 4)
        self.grad = z(1, 4)          # the last reduced gradient (ngp_intrinsics_adam's grad_out)
        self.grad_rays = z(0, 4)     # one row per ray of the current batch
        self.flag = z(1, dtype=torch.int32)   # non-invertible pixels of the module path's directions()
        self.n_rays = 0
        self.pix = self.dirs = None

    def reserve(self, n: int):
        """Make the per-ray gradient buffer hold n rays (before a graph captures it)."""
        if self.grad_rays.shape[0] < n:
            self.grad_rays = torch.zeros(n, 4, device=self.poses.device)
        return self.grad_rays

    def directions(self, pix_idxs, out=None, found_inf=None):
        """Directions [n, 3] of the pixels pix_idxs [n] int64 under the current corrections; starts a batch (its
        gradient rows are cleared).  A pixel that is not invertible raises ``found_inf`` (default: the flag the
        trainer folds into its own at the update)."""
        pix = pix_idxs.to(torch.int64).reshape(-1).contiguous()
        n = pix.numel()
        self.reserve(n)
        self.n_rays, self.pix = n, pix
        self.dirs = ops.camera_unproject(self.camera, self.W, self.H, pix, self.corr, out=out,
                                         grad_rows=self.grad_rays[:n],
                                         found_inf=self.flag if found_inf is None else found_inf)
        return self.dirs

    def table(self):
        """Directions [W*H, 3] of every pixel under the current corrections (test views of the training camera)."""
        return ops.camera_unproject(self.camera, self.W, self.H, corr=self.corr, device=self.poses.device)

    def accumulate(self, dx, ts, rays_a, img_idxs, pose_corr=None, n_rays_dev=None, found_inf=None):
        """The per-ray gradient rows of the batch of the last directions() call from its sample gradients dx."""
        ops.intrinsics_grad(dx, ts, rays_a, self.pix, img_idxs, self.poses, self.dirs, self.camera, self.W, self.H,
                            self.corr, self.grad_rays[:self.n_rays], pose_corr=pose_corr, n_rays_dev=n_rays_dev,
                            found_inf=found_inf)

    def enqueue_adam(self, trainer):
        """Reduce the batch's rows and take the corrections' Adam step on the trainer's device scalars."""
        ops.intrinsics_adam(self.corr, self.grad_rays, self.n_rays, self.exp_avg, self.exp_avg_sq, trainer.hyper,
                            self.lr_ratio, found_inf=trainer.found_inf, beta1=trainer.betas[0],
                            beta2=trainer.betas[1], eps=trainer.eps, grad_out=self.grad)

    def state(self):
        return [self.corr, self.exp_avg, self.exp_avg_sq, self.grad, self.grad_rays, self.flag]

    def refined(self):
        """(fx', fy', cx', cy') in fp64 under the current corrections."""
        a, bx, by, _ = (float(v) for v in self.corr.detach().cpu().numpy()[0])
        c = self.camera
        e = math.exp(a)
        return c.fx * e, c.fy * e, c.cx + self.W * bx, c.cy + self.H * by

    def refined_camera(self) -> Camera:
        fx, fy, cx, cy = self.refined()
        return dataclasses.replace(self.camera, fx=fx, fy=fy, cx=cx, cy=cy)
