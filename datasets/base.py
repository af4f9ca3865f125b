"""``BaseDataset`` of the disk loaders (reference datasets/base.py:6-61): length, ``to(device)`` and batch sampling.

A training split's ``dataset[idx]`` draws ``batch_size`` rays with ``torch.randint`` on the rays' device:
'all_images' draws an image per ray, 'same_image' takes every ray from image ``idx``; both then draw the pixels.
Other splits return the pose of view ``idx`` and, when the split has images, its colours.

``rays`` is [N, H*W, 3], or [N, H*W, 4] when an image had an alpha channel: the fourth column is the resized alpha,
and ``rgb`` (the reference's value) stays ``rays[..., :3]``; samples then also carry ``alpha``.  ``bg_load`` is the
colour the loader blended transparent pixels onto (1 white, 0 black), which ``--random_bg`` replaces.

A loader that reads depth (the ngp loader's ``depth_path``, DESIGN.md §6h) sets ``depths`` [N, H*W] fp32 z-depth, 0
where there is none; samples then also carry ``depth``, indexed as ``rgb`` is.  Loaders without depth set nothing and
their samples are unchanged.

A loader built with ``lens_distortion=True`` (DESIGN.md §6l) sets ``camera`` (taichi_nerfs_b200.intrinsics.Camera);
``to(device)`` then replaces ``directions`` by the unprojection of every pixel through it, on the GPU, and raises if
a pixel is not invertible.  Loaders without it have ``camera = None`` and keep the pinhole ``directions``.
"""
from __future__ import annotations

import numpy as np
import torch
from torch.utils.data import Dataset


def stack_images(imgs):
    """[N, H*W, C] float32 tensor of the loaded images; when some have an alpha column, the rest get alpha 1."""
    if not imgs:
        return torch.empty(0)
    if any(i.shape[1] == 4 for i in imgs):
        imgs = [i if i.shape[1] == 4 else np.concatenate([i, np.ones_like(i[:, :1])], 1) for i in imgs]
    return torch.from_numpy(np.stack(imgs).astype(np.float32, copy=False))


def stack_poses(poses):
    """[N, 3, 4] float32 from float64 camera-to-world matrices (one rounding, as torch.FloatTensor(list) does)."""
    return torch.from_numpy(np.asarray(poses, dtype=np.float64).reshape(-1, 3, 4).astype(np.float32))


class BaseDataset(Dataset):
    bg_load = 1.0
    camera = None

    def __init__(self, root_dir, split='train', downsample=1.0):
        self.root_dir = root_dir
        self.split = split
        self.downsample = downsample
        self.batch_size = 8192
        self.ray_sampling_strategy = 'all_images'

    def read_intrinsics(self):
        raise NotImplementedError

    def __len__(self):
        return len(self.poses)

    def to(self, device):
        self.rays = self.rays.to(device)
        self.poses = self.poses.to(device)
        self.K = self.K.to(device)
        self.directions = self.directions.to(device)
        if self.camera is not None:
            from taichi_nerfs_b200.intrinsics import unproject_table
            self.directions = unproject_table(self.camera, *self.img_wh, self.directions.device)
        if getattr(self, 'depths', None) is not None:
            self.depths = self.depths.to(device)
        return self

    def gather(self, img_idxs, pix_idxs):
        """The training sample of the rays (img_idxs[i], pix_idxs[i]): the dict a training split's ``dataset[idx]``
        returns for those indices (``img_idxs`` may be one index for the whole batch, as 'same_image' gives)."""
        rays = self.rays[img_idxs, pix_idxs]
        sample = {'img_idxs': img_idxs, 'pix_idxs': pix_idxs, 'pose': self.poses[img_idxs],
                  'direction': self.directions[pix_idxs], 'rgb': rays[:, :3]}
        if getattr(self, 'depths', None) is not None:
            sample['depth'] = self.depths[img_idxs, pix_idxs]
        if rays.shape[-1] == 4:
            sample['alpha'] = rays[:, 3]
        return sample

    def __getitem__(self, idx):
        if self.split.startswith('train'):
            dev = self.rays.device
            if self.ray_sampling_strategy == 'all_images':
                img_idxs = torch.randint(0, len(self.poses), size=(self.batch_size,), device=dev)
            elif self.ray_sampling_strategy == 'same_image':
                img_idxs = [idx]
            else:
                raise ValueError(f"unknown ray_sampling_strategy {self.ray_sampling_strategy!r}")
            pix_idxs = torch.randint(0, self.img_wh[0] * self.img_wh[1], size=(self.batch_size,), device=dev)
            return self.gather(img_idxs, pix_idxs)
        else:
            sample = {'pose': self.poses[idx], 'img_idxs': idx}
            if len(self.rays) > 0:
                rays = self.rays[idx]
                sample['rgb'] = rays[:, :3]
                if getattr(self, 'depths', None) is not None:
                    sample['depth'] = self.depths[idx]
            else:
                return sample
        if rays.shape[-1] == 4:
            sample['alpha'] = rays[:, 3]
        return sample
