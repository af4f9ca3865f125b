"""fp64 restatement of the camera model of DESIGN.md §6l (csrc/camera.cu) in torch, for the intrinsics tests.

Newton's method is unrolled over a fixed number of iterations, so torch.autograd differentiates the undistorted
coordinates with respect to the intrinsics corrections, and the whole ray with respect to them through Rodrigues.
"""
from __future__ import annotations

import numpy as np
import torch

NEWTON_ITERS = 20


def distort(dist, x, y):
    """D(x, y) of the OPENCV form with dist = (k1, k2, p1, p2)."""
    k1, k2, p1, p2 = dist
    r2 = x * x + y * y
    rad = 1.0 + k1 * r2 + k2 * r2 * r2
    return (x * rad + 2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x),
            y * rad + p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y)


def jacobian(dist, x, y):
    """J_D (j00, j01, j10, j11) in closed form."""
    k1, k2, p1, p2 = dist
    r2 = x * x + y * y
    rad = 1.0 + k1 * r2 + k2 * r2 * r2
    q = 2.0 * k1 + 4.0 * k2 * r2
    j01 = q * x * y + 2.0 * p1 * x + 2.0 * p2 * y
    return (rad + q * x * x + 2.0 * p1 * y + 6.0 * p2 * x, j01, j01, rad + q * y * y + 6.0 * p1 * y + 2.0 * p2 * x)


def undistort(dist, xd, yd, iters=NEWTON_ITERS):
    """U(x_d, y_d) by unrolled Newton from (x_d, y_d) (differentiable)."""
    x, y = xd, yd
    for _ in range(iters):
        fx, fy = distort(dist, x, y)
        fx, fy = fx - xd, fy - yd
        a, b, c, d = jacobian(dist, x, y)
        det = a * d - b * c
        x, y = x - (d * fx - b * fy) / det, y - (a * fy - c * fx) / det
    return x, y


def pixel_xd(pix, W, H, fx, fy, cx, cy, corr=None):
    """(x_d, y_d) fp64 of pixels pix under corrections corr = (a, b_x, b_y) (tensors, differentiable)."""
    pix = torch.as_tensor(pix, dtype=torch.int64)
    u, v = (pix % W).double(), torch.div(pix, W, rounding_mode='floor').double()
    if corr is not None:
        e = torch.exp(corr[0])
        fx, fy, cx, cy = fx * e, fy * e, cx + W * corr[1], cy + H * corr[2]
    return (u - cx + 0.5) / fx, (v - cy + 0.5) / fy


def so3_exp(w):
    """Exp of one rotation vector w [3] (torch fp64, differentiable; w = 0 gives I)."""
    t2 = (w * w).sum()
    K = torch.zeros(3, 3, dtype=w.dtype)
    K = K.index_put((torch.tensor([0, 0, 1, 1, 2, 2]), torch.tensor([1, 2, 0, 2, 0, 1])),
                    torch.stack([-w[2], w[1], w[2], -w[0], -w[1], w[0]]))
    if float(t2) < 1e-6:
        A, B = 1 - t2 / 6 + t2 * t2 / 120, 0.5 - t2 / 24 + t2 * t2 / 720
    else:
        t = torch.sqrt(t2)
        A, B = torch.sin(t) / t, 2 * torch.sin(t / 2) ** 2 / t2
    return torch.eye(3, dtype=w.dtype) + A * K + B * (K @ K)


def border_pixels(W, H):
    u, v = np.arange(W), np.arange(H)
    return np.unique(np.concatenate([u, (H - 1) * W + u, v * W, v * W + W - 1])).astype(np.int64)
