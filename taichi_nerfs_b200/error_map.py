"""Error-map ray sampling (``--ray_sampling_strategy error_map``, DESIGN.md §6j): training pixels are drawn in
proportion to their recent error.

Every training image is cut into ``res x res`` tiles (clamped to min(W, H)).  Each tile keeps an integer EMA of the
squared colour error of the rays drawn in it (fixed point 2^30).  Every step's rays add their errors to the tiles
(``accumulate``); every density-grid update folds them into the EMA and rebuilds the sampling CDF (``rebuild``).  A
pixel is drawn with probability proportional to its tile's error plus a floor, so every pixel keeps probability at
least ``floor / N_pix``.  Each drawn ray carries the weight w = 1 / (N_pix p(pixel)) <= 1 / floor: scaling a ray's
loss by w makes the expected loss the uniform one.  With a uniform map every weight is exactly 1.0.

All arithmetic of the map is integer (csrc/errmap.cu): the map, its CDF and the draws are bit-reproducible.
"""
from __future__ import annotations

from fractions import Fraction

import torch

from . import ops
from ._lib import load

FIXED_ONE = 1 << 30      # fixed-point 1.0 of the per-tile error
# starting error of every tile: 0, so the map starts uniform and a tile no ray has reached yet is drawn through the floor
# only (a high prior keeps unvisited background tiles in the draws for hundreds of steps)
INIT_ERROR = 0
# the counter word of the draws (csrc/errmap.cu kErrMapCounterWord)
COUNTER_WORD = 0x656D0001


def floor_fraction(floor: float):
    """(p, q) with p / q the floor as a fraction of denominator <= 1024."""
    f = Fraction(float(floor)).limit_denominator(1024)
    if not 0 < f < 1:
        raise ValueError(f"error map: floor must be in (0, 1), got {floor}")
    return f.numerator, f.denominator


class ErrorMap:
    """Per-tile error map of ``n_img`` training images of ``W x H`` pixels on one device."""

    def __init__(self, n_img: int, W: int, H: int, res: int = 64, ema_shift: int = 2, floor: float = 0.2,
                 seed: int = 0, device=None):
        n_img, W, H, res = int(n_img), int(W), int(H), int(res)
        if n_img <= 0 or W <= 0 or H <= 0:
            raise ValueError(f"error map: need images, got {n_img} of {W}x{H}")
        if res < 1:
            raise ValueError(f"error map: res must be >= 1, got {res}")
        if not 0 <= int(ema_shift) < 32:
            raise ValueError(f"error map: ema_shift must be in [0, 32), got {ema_shift}")
        self.R = min(res, W, H)
        self.geom = (n_img, W, H, self.R)
        self.n_img, self.W, self.H = n_img, W, H
        self.T = n_img * self.R * self.R
        self.n_pix = n_img * W * H
        self.ema_shift = int(ema_shift)
        self.floor_num, self.floor_den = floor_fraction(floor)
        self.seed = int(seed)
        dev = torch.device("cuda") if device is None else torch.device(device)
        self.E = torch.full((self.T,), INIT_ERROR, device=dev, dtype=torch.int64)
        self.acc = torch.zeros(self.T, device=dev, dtype=torch.int64)
        self.cnt = torch.zeros(self.T, device=dev, dtype=torch.int32)
        self.cdf = torch.zeros(self.T, device=dev, dtype=torch.int64)
        ws = int(load().ngp_error_map_workspace_bytes(self.T))
        self.workspace = torch.zeros((ws + 7) // 8, device=dev, dtype=torch.int64)
        self.rebuild()

    @property
    def max_weight(self) -> float:
        return self.floor_den / self.floor_num

    def draw(self, n: int, step: int = 0, step_dev=None, out=None):
        """(img_idxs [n] int64, pix_idxs [n] int64, w [n] fp32) of training step ``step`` (or step_dev[0])."""
        return ops.error_map_sample(self.cdf, self.geom, n, self.seed, step=step, step_dev=step_dev, out=out)

    def accumulate(self, pred, target, img_idxs, pix_idxs, bg_rgb=None, alpha=None, b_load=1.0):
        """Add the rays' errors sum_c (pred - target)^2 to their tiles; with ``bg_rgb`` and ``alpha`` the target is the
        random-background one, target + (bg_rgb - b_load)(1 - alpha)."""
        ops.error_map_accumulate(pred, target, img_idxs, pix_idxs, self.geom, self.acc, self.cnt, bg_rgb=bg_rgb,
                                 alpha=alpha, b_load=b_load)

    def rebuild(self):
        """Fold the accumulated errors into the EMA and rebuild the sampling CDF."""
        ops.error_map_rebuild(self.E, self.acc, self.cnt, self.cdf, self.geom, self.ema_shift, self.floor_num,
                              self.floor_den, self.workspace)

    def as_image(self):
        """fp32 [n_img, R, R] per-tile error E / 2^30."""
        return (self.E.to(torch.float64) / FIXED_ONE).to(torch.float32).reshape(self.n_img, self.R, self.R)

    def state(self):
        return [self.E, self.acc, self.cnt, self.cdf]
