"""Camera-ray helpers — mirrors get_ray_directions / get_rays of the reference's
datasets/ray_utils.py (:8-48, :51-80) without the kornia dependency.  fp32 even under autocast.  The pose helpers
of the COLMAP loader (average_poses, center_poses, create_spheric_poses) follow :118-221 in float64."""
from __future__ import annotations

import numpy as np
import torch


@torch.amp.autocast('cuda', enabled=False)
def get_ray_directions(H, W, K, device='cpu', random=False, return_uv=False, flatten=True):
    """Per-pixel directions in the camera frame [right, down, front]: ((u-cx+.5)/fx, (v-cy+.5)/fy, 1)."""
    v, u = torch.meshgrid(torch.arange(H, device=device, dtype=torch.float32),
                          torch.arange(W, device=device, dtype=torch.float32), indexing='ij')
    grid = torch.stack([u, v], dim=-1)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    if random:
        du, dv = torch.rand_like(u), torch.rand_like(v)
    else:
        du = dv = 0.5
    directions = torch.stack([(u - cx + du) / fx, (v - cy + dv) / fy, torch.ones_like(u)], -1)
    if flatten:
        directions = directions.reshape(-1, 3)
        grid = grid.reshape(-1, 2)
    if return_uv:
        return directions, grid
    return directions


@torch.amp.autocast('cuda', enabled=False)
def get_rays(directions, c2w):
    """World-space origins / (un-normalised) directions for camera-frame ``directions`` (N,3) and a
    camera-to-world matrix (3,4) or per-ray matrices (N,3,4)."""
    if c2w.ndim == 2:
        rays_d = directions @ c2w[:, :3].T
    else:
        rays_d = torch.einsum('nc,nac->na', directions, c2w[..., :3])
    rays_o = c2w[..., 3].expand_as(rays_d)
    return rays_o, rays_d


def normalize(v):
    return v / np.linalg.norm(v)


def average_poses(poses, pts3d=None):
    """(3,4) average pose of (N,3,4) ``poses`` (reference ray_utils.py:118-157): centre = mean of ``pts3d`` (of the
    camera positions without it); z = normalised mean z axis; x = normalise(mean y axis × z); y = z × x."""
    center = pts3d.mean(0) if pts3d is not None else poses[..., 3].mean(0)
    z = normalize(poses[..., 2].mean(0))
    x = normalize(np.cross(poses[..., 1].mean(0), z))
    y = np.cross(z, x)
    return np.stack([x, y, z, center], 1)


def center_poses(poses, pts3d=None):
    """Poses (and points) expressed in the frame of ``average_poses`` (reference ray_utils.py:160-190), float64."""
    avg = np.eye(4)
    avg[:3] = average_poses(poses, pts3d)
    avg_inv = np.linalg.inv(avg)
    bottom = np.tile(np.array([0, 0, 0, 1]), (len(poses), 1, 1))
    centered = (avg_inv @ np.concatenate([poses, bottom], 1))[:, :3]
    if pts3d is None:
        return centered
    return centered, pts3d @ avg_inv[:, :3].T + avg_inv[:, 3:].T


def create_spheric_poses(radius, mean_h, n_poses=120):
    """(n_poses,3,4) cameras on a circle about the z axis at elevation -15° (reference ray_utils.py:193-221): for
    each azimuth θ, c2w = P · R_y(θ) · R_x(-π/12) · T(radius) with T translating by (0, 2·mean_h, -radius) and P the
    fixed axis permutation [[-1,0,0],[0,0,1],[0,1,0]]."""
    def rot_x(phi):
        return np.array([[1, 0, 0], [0, np.cos(phi), -np.sin(phi)], [0, np.sin(phi), np.cos(phi)]])

    def rot_y(th):
        return np.array([[np.cos(th), 0, -np.sin(th)], [0, 1, 0], [np.sin(th), 0, np.cos(th)]])

    trans = np.array([[1, 0, 0, 0], [0, 1, 0, 2 * mean_h], [0, 0, 1, -radius]])
    perm = np.array([[-1, 0, 0], [0, 0, 1], [0, 1, 0]])
    out = [perm @ (rot_y(th) @ rot_x(-np.pi / 12) @ trans)
           for th in np.linspace(0, 2 * np.pi, n_poses + 1)[:-1]]
    return np.stack(out, 0)
