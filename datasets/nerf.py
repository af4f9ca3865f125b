"""Blender-layout loader (``transforms_{split}.json`` + ``{file_path}.png``; reference datasets/nerf.py).

- Intrinsics (:23-36): 800x800 scaled by ``downsample``, focal ``0.5 * 800 / tan(0.5 * camera_angle_x)``.
- Poses (:54-62): ``transform_matrix[:3, :4]`` with the y and z axes negated ([right up back] -> [right down front])
  and the camera position rescaled to radius 1.5, in float64 until the final cast.
- ``trainval`` (:42-49) reads the train and then the val frames.
- Images (:64-70) are blended onto white.  In a test or val split a frame whose image file is missing keeps its pose
  (the reference skips the image and keeps the pose too); a training split with a missing image is refused, since
  its rays would be paired with the wrong poses.  Any other failure to read an image raises, where the reference
  ignores it.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from .base import BaseDataset, stack_images, stack_poses
from .color_utils import read_image
from .ray_utils import get_ray_directions


class NeRFDataset(BaseDataset):
    bg_load = 1.0

    def __init__(self, root_dir, split='train', downsample=1.0, read_meta=True, **_):
        super().__init__(root_dir, split, downsample)
        self.read_intrinsics()
        if read_meta:
            self.read_meta(split)

    def _frames(self, name):
        with open(os.path.join(self.root_dir, f"transforms_{name}.json")) as f:
            return json.load(f)

    def read_intrinsics(self):
        meta = self._frames('train')
        w = h = int(800 * self.downsample)
        fx = fy = 0.5 * 800 / np.tan(0.5 * meta['camera_angle_x']) * self.downsample
        self.K = torch.from_numpy(np.float32([[fx, 0, w / 2], [0, fy, h / 2], [0, 0, 1]]))
        self.directions = get_ray_directions(h, w, self.K)
        self.img_wh = (w, h)

    def read_meta(self, split):
        if split == 'trainval':
            frames = self._frames('train')['frames'] + self._frames('val')['frames']
        else:
            frames = self._frames(split)['frames']
        poses, imgs = [], []
        for frame in frames:
            c2w = np.array(frame['transform_matrix'], dtype=np.float64)[:3, :4]
            c2w[:, 1:3] *= -1
            c2w[:, 3] /= np.linalg.norm(c2w[:, 3]) / 1.5
            poses.append(c2w)
            path = os.path.join(self.root_dir, f"{frame['file_path']}.png")
            if os.path.exists(path):
                imgs.append(read_image(path, self.img_wh, keep_alpha=True))
        if split.startswith('train') and len(imgs) != len(poses):
            raise ValueError(f"{self.root_dir}: {len(poses) - len(imgs)} of the {len(poses)} {split} frames have no "
                             "image; a training split needs every image (rays and poses are sampled by index)")
        self.rays = stack_images(imgs)
        self.poses = stack_poses(poses)
