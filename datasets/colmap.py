"""COLMAP-layout loader (``sparse/0/{cameras,images,points3D}.bin`` + an image folder; reference
datasets/colmap.py without its HDR-NeRF branches, whose exposure channel the reference's training never reads).

- Intrinsics (:25-47) come from camera 1: ``SIMPLE_RADIAL`` (f, cx, cy, k: distortion ignored), ``PINHOLE`` and
  ``OPENCV`` (fx, fy, cx, cy, ...: distortion ignored), scaled by ``downsample``.  Other models are refused by name.
  With ``lens_distortion=True`` (DESIGN.md §6l) the distortion is kept: ``camera`` holds the model (``PINHOLE``,
  ``SIMPLE_PINHOLE``, ``SIMPLE_RADIAL``, ``RADIAL`` or ``OPENCV``; others are refused by name) with its focal lengths and
  principal point scaled and its distortion terms as written, and ``to(device)`` unprojects every pixel through it.
- Poses (:49-87): images sorted by name; camera-to-world = inverse of the world-to-camera matrix in float64;
  recentred on the average pose about the sparse points' mean (``center_poses``) and scaled so that the nearest
  camera is at distance 1.
- Splits (:141-150): ``test`` is every 8th image, ``train`` the rest, any other split all images.  ``test_traj``
  (:89-94) is 120 poses on a circle (``create_spheric_poses``) and no images.
- Images come from ``images_{1/downsample}`` for a ``360_v2`` path with ``downsample < 1`` (:56-59), else
  ``images``; their alpha, if any, is premultiplied (onto black).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .base import BaseDataset, stack_images, stack_poses
from .color_utils import read_image
from .colmap_model import read_cameras_binary, read_images_binary, read_points3d_binary
from .ray_utils import center_poses, create_spheric_poses, get_ray_directions


class ColmapDataset(BaseDataset):
    bg_load = 0.0

    def __init__(self, root_dir, split='train', downsample=1.0, read_meta=True, lens_distortion=False, **_):
        if 'HDR-NeRF' in root_dir:
            raise ValueError(f"{root_dir}: HDR-NeRF data (multi-exposure images) is not supported by the COLMAP loader")
        super().__init__(root_dir, split, downsample)
        self.lens_distortion = bool(lens_distortion)
        self.read_intrinsics()
        if read_meta:
            self.read_meta(split)

    def read_intrinsics(self):
        cams = read_cameras_binary(os.path.join(self.root_dir, 'sparse/0/cameras.bin'))
        if 1 not in cams:
            raise ValueError(f"{self.root_dir}: sparse/0/cameras.bin has no camera with id 1")
        cam = cams[1]
        h, w = int(cam.height * self.downsample), int(cam.width * self.downsample)
        self.img_wh = (w, h)
        p = cam.params
        if self.lens_distortion:
            self._read_camera(cam.model, p, w, h)
            return
        if cam.model == 'SIMPLE_RADIAL':
            fx = fy = p[0] * self.downsample
            cx, cy = p[1] * self.downsample, p[2] * self.downsample
        elif cam.model in ('PINHOLE', 'OPENCV'):
            fx, fy = p[0] * self.downsample, p[1] * self.downsample
            cx, cy = p[2] * self.downsample, p[3] * self.downsample
        else:
            raise ValueError(f"camera model {cam.model} is not supported (SIMPLE_RADIAL, PINHOLE, OPENCV are)")
        self.K = torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=torch.float32)
        self.directions = get_ray_directions(h, w, self.K)

    def _read_camera(self, model, p, w, h):
        from taichi_nerfs_b200.intrinsics import Camera
        d = self.downsample
        if model in ('SIMPLE_PINHOLE', 'SIMPLE_RADIAL', 'RADIAL'):   # f, cx, cy[, k1[, k2]]
            f, cx, cy, dist = p[0] * d, p[1] * d, p[2] * d, list(p[3:])
            self.camera = Camera(model, f, f, cx, cy, tuple(dist + [0.0] * (4 - len(dist))))
        elif model in ('PINHOLE', 'OPENCV'):                          # fx, fy, cx, cy[, k1, k2, p1, p2]
            dist = list(p[4:])
            self.camera = Camera(model, p[0] * d, p[1] * d, p[2] * d, p[3] * d, tuple(dist + [0.0] * (4 - len(dist))))
        else:
            raise ValueError(f"camera model {model} is not supported with lens distortion (PINHOLE, SIMPLE_PINHOLE, "
                             f"SIMPLE_RADIAL, RADIAL, OPENCV are)")
        self.K = self.camera.K()
        self.directions = get_ray_directions(h, w, self.K)   # the pinhole table until to(device) unprojects

    def read_meta(self, split):
        imdata = read_images_binary(os.path.join(self.root_dir, 'sparse/0/images.bin'))
        names = [im.name for im in imdata.values()]
        perm = np.argsort(names)
        if '360_v2' in self.root_dir and self.downsample < 1:
            folder = f'images_{int(1 / self.downsample)}'
        else:
            folder = 'images'
        img_paths = [os.path.join(self.root_dir, folder, n) for n in sorted(names)]
        bottom = np.array([[0, 0, 0, 1.]])
        w2c = np.stack([np.concatenate([np.concatenate([im.qvec2rotmat(), im.tvec.reshape(3, 1)], 1), bottom], 0)
                        for im in imdata.values()])
        poses = np.linalg.inv(w2c)[perm, :3]
        pts = read_points3d_binary(os.path.join(self.root_dir, 'sparse/0/points3D.bin'))
        pts3d = np.array([p.xyz for p in pts.values()])
        poses, self.pts3d = center_poses(poses, pts3d)
        scale = np.linalg.norm(poses[..., 3], axis=-1).min()
        poses[..., 3] /= scale
        self.pts3d /= scale

        if split == 'test_traj':
            ring = poses[::8]
            self.poses = stack_poses(create_spheric_poses(1.2, ring[:, 1, 3].mean()))
            self.rays = torch.empty(0)
            return
        if split == 'train':
            keep = [i for i in range(len(img_paths)) if i % 8 != 0]
        elif split == 'test':
            keep = [i for i in range(len(img_paths)) if i % 8 == 0]
        else:
            keep = list(range(len(img_paths)))
        self.rays = stack_images([read_image(img_paths[i], self.img_wh, blend_a=False, keep_alpha=True)
                                  for i in keep])
        self.poses = stack_poses(poses[keep])
