"""instant-ngp-layout loader (one ``transforms.json`` with ``w``, ``h``, ``fl_x``, ``fl_y`` and the frames;
reference datasets/ngp.py).  Every split reads all frames (:43-72), as the reference does.

- Intrinsics (:22-41): ``w``, ``h``, ``fl_x``, ``fl_y`` scaled by ``downsample``, principal point at the centre.
- Poses (:64-66): ``transform_matrix[:3, :4]`` with the y and z axes negated; no rescaling.
- A frame whose image file (``file_path`` as written, extension included) is missing is skipped, pose and all.
- Images are blended onto white.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from .base import BaseDataset, stack_images, stack_poses
from .color_utils import read_image
from .ray_utils import get_ray_directions


class NGPDataset(BaseDataset):
    bg_load = 1.0

    def __init__(self, root_dir, split='train', downsample=1.0, read_meta=True, **_):
        super().__init__(root_dir, split, downsample)
        self.read_intrinsics()
        if read_meta:
            self.read_meta(split)

    def _meta(self):
        with open(os.path.join(self.root_dir, "transforms.json")) as f:
            return json.load(f)

    def read_intrinsics(self):
        meta = self._meta()
        w, h = int(meta['w'] * self.downsample), int(meta['h'] * self.downsample)
        fx, fy = meta['fl_x'] * self.downsample, meta['fl_y'] * self.downsample
        self.K = torch.from_numpy(np.float32([[fx, 0, w / 2], [0, fy, h / 2], [0, 0, 1]]))
        self.directions = get_ray_directions(h, w, self.K)
        self.img_wh = (w, h)

    def read_meta(self, split):
        poses, imgs = [], []
        for frame in self._meta()['frames']:
            path = os.path.join(self.root_dir, f"{frame['file_path']}")
            if not os.path.exists(path):
                continue
            imgs.append(read_image(path, self.img_wh, keep_alpha=True))
            c2w = np.array(frame['transform_matrix'], dtype=np.float64)[:3, :4]
            c2w[:, 1:3] *= -1
            poses.append(c2w)
        self.rays = stack_images(imgs)
        self.poses = stack_poses(poses)
