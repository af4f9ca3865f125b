"""NSVF-layout loader (``intrinsics.txt``, ``bbox.txt``, ``rgb/{0,1,2}_*.png``, ``pose/{0,1,2}_*.txt``; reference
datasets/nsvf.py).  Which branch applies depends on the directory name, as in the reference.

- Bounds (:20-33): ``bbox.txt``'s first six numbers are (xyz_min, xyz_max); shift = their midpoint, scale = half
  the largest extent x 1.05, then x 1.2 for a path containing ``Mic``, else x 1.1 for one containing ``Lego``.
  Camera positions become ``(p - shift) / (2 scale)``: the scene fits in [-0.5, 0.5]^3.
- Intrinsics (:35-56): ``Synthetic`` (800x800) and ``Ignatius`` (1920x1080) read one focal length from the first
  line of ``intrinsics.txt``; ``BlendedMVS`` (768x576) and ``Tanks`` (1920x1080) read a 3x3 (or 4x4) matrix.  All
  scale by ``downsample``.  A directory matching none of the four names is refused (the reference fails later
  with a NameError).
- Splits (:78-92): ``train`` '0_', ``trainval`` '0_' and '1_', ``trainvaltest`` '0_' to '2_', ``val`` '1_'; any
  other split is '2_' for ``Synthetic`` and, otherwise, ``test`` is '1_'.  ``test_traj`` (:62-76) reads poses only,
  from ``test_pose/*.txt`` (``Ignatius``) or ``test_traj.txt``, with the x axis negated.
- Images are blended onto white.  For ``Jade`` and ``Fountain``, whose backgrounds are black, pixels whose three
  colour channels are all <= 0.1 become 1.0.  That is the intent of the reference's line (:109-111), which mixes
  ``torch.all`` with a numpy array and fails.
"""
from __future__ import annotations

import glob
import os

import numpy as np
import torch

from .base import BaseDataset, stack_images, stack_poses
from .color_utils import read_image
from .ray_utils import get_ray_directions


class NSVFDataset(BaseDataset):
    bg_load = 1.0

    def __init__(self, root_dir, split='train', downsample=1.0, **kwargs):
        super().__init__(root_dir, split, downsample)
        self.read_intrinsics()
        if kwargs.get('read_meta', True):
            xyz_min, xyz_max = np.loadtxt(os.path.join(root_dir, 'bbox.txt'))[:6].reshape(2, 3)
            self.shift = (xyz_max + xyz_min) / 2
            self.scale = (xyz_max - xyz_min).max() / 2 * 1.05
            if 'Mic' in self.root_dir:
                self.scale *= 1.2
            elif 'Lego' in self.root_dir:
                self.scale *= 1.1
            self.read_meta(split)

    def read_intrinsics(self):
        path = os.path.join(self.root_dir, 'intrinsics.txt')
        if 'Synthetic' in self.root_dir or 'Ignatius' in self.root_dir:
            with open(path) as f:
                fx = fy = float(f.readline().split()[0]) * self.downsample
            if 'Synthetic' in self.root_dir:
                w = h = int(800 * self.downsample)
            else:
                w, h = int(1920 * self.downsample), int(1080 * self.downsample)
            K = np.float32([[fx, 0, w / 2], [0, fy, h / 2], [0, 0, 1]])
        else:
            if 'BlendedMVS' in self.root_dir:
                w, h = int(768 * self.downsample), int(576 * self.downsample)
            elif 'Tanks' in self.root_dir:
                w, h = int(1920 * self.downsample), int(1080 * self.downsample)
            else:
                raise ValueError(f"{self.root_dir}: the NSVF loader picks the image size from the directory name, "
                                 "which must contain Synthetic, Ignatius, BlendedMVS or Tanks")
            K = np.loadtxt(path, dtype=np.float32)[:3, :3]
            K[:2] *= self.downsample
        self.K = torch.from_numpy(np.ascontiguousarray(K))
        self.directions = get_ray_directions(h, w, self.K)
        self.img_wh = (w, h)

    def _to_unit_box(self, c2w):
        c2w[:, 3] -= self.shift
        c2w[:, 3] /= 2 * self.scale
        return c2w

    def read_meta(self, split):
        poses, imgs = [], []
        if split == 'test_traj':
            if 'Ignatius' in self.root_dir:
                raw = [np.loadtxt(p) for p in sorted(glob.glob(os.path.join(self.root_dir, 'test_pose/*.txt')))]
            else:
                raw = np.loadtxt(os.path.join(self.root_dir, 'test_traj.txt')).reshape(-1, 4, 4)
            for pose in raw:
                c2w = pose[:3]
                c2w[:, 0] *= -1  # [left down front] to [right down front]
                poses.append(self._to_unit_box(c2w))
        else:
            if split == 'train':
                prefix = '0_'
            elif split == 'trainval':
                prefix = '[0-1]_'
            elif split == 'trainvaltest':
                prefix = '[0-2]_'
            elif split == 'val':
                prefix = '1_'
            elif 'Synthetic' in self.root_dir:
                prefix = '2_'
            elif split == 'test':
                prefix = '1_'
            else:
                raise ValueError(f'{split} split not recognized!')
            img_paths = sorted(glob.glob(os.path.join(self.root_dir, 'rgb', prefix + '*.png')))
            pose_paths = sorted(glob.glob(os.path.join(self.root_dir, 'pose', prefix + '*.txt')))
            black_bg = 'Jade' in self.root_dir or 'Fountain' in self.root_dir
            for img_path, pose_path in zip(img_paths, pose_paths):
                poses.append(self._to_unit_box(np.loadtxt(pose_path)[:3]))
                img = read_image(img_path, self.img_wh, keep_alpha=True)
                if black_bg:
                    img[np.all(img[:, :3] <= 0.1, axis=-1), :3] = 1.0
                imgs.append(img)
        self.rays = stack_images(imgs)
        self.poses = stack_poses(poses)
