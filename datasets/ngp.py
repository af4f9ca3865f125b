"""instant-ngp-layout loader (one ``transforms.json`` with ``w``, ``h``, ``fl_x``, ``fl_y`` and the frames;
reference datasets/ngp.py).  Every split reads all frames (:43-72), as the reference does.

- Intrinsics (:22-41): ``w``, ``h``, ``fl_x``, ``fl_y`` scaled by ``downsample``, principal point at the centre.
  With ``lens_distortion=True`` (DESIGN.md §6l) ``cx``, ``cy`` are read when present (scaled) and ``k1 k2 p1 p2`` as
  an OPENCV ``camera`` (unscaled), and ``to(device)`` unprojects every pixel through it; ``is_fisheye`` and non-zero
  ``k3`` / ``k4`` are refused.
- Poses (:64-66): ``transform_matrix[:3, :4]`` with the y and z axes negated; no rescaling.
- A frame whose image file (``file_path`` as written, extension included) is missing is skipped, pose and all.
- Images are blended onto white.
- Depth (DESIGN.md §6h): when any frame has ``depth_path``, ``depths`` [n_img, H*W] fp32 holds z-depth =
  pixel value x the top-level ``integer_depth_scale`` (instant-ngp's RGB-D convention; required then).  The depth
  image is a single-channel integer PNG of the json's ``w`` x ``h``, read with PIL and downsampled by nearest neighbour
  (never averaged across a depth edge).  A frame without ``depth_path`` gets zeros ("no depth"); a skipped frame drops
  its depth with its image.  Without any ``depth_path`` there is no ``depths`` attribute.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch
from PIL import Image

from .base import BaseDataset, stack_images, stack_poses
from .color_utils import read_image
from .ray_utils import get_ray_directions


class NGPDataset(BaseDataset):
    bg_load = 1.0

    def __init__(self, root_dir, split='train', downsample=1.0, read_meta=True, lens_distortion=False, **_):
        super().__init__(root_dir, split, downsample)
        self.lens_distortion = bool(lens_distortion)
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
        if self.lens_distortion:
            self._read_camera(meta, fx, fy, w, h)
            return
        self.K = torch.from_numpy(np.float32([[fx, 0, w / 2], [0, fy, h / 2], [0, 0, 1]]))
        self.directions = get_ray_directions(h, w, self.K)
        self.img_wh = (w, h)

    def _read_camera(self, meta, fx, fy, w, h):
        from taichi_nerfs_b200.intrinsics import Camera
        where = f"{self.root_dir}/transforms.json"
        if meta.get('is_fisheye', False):
            raise ValueError(f"{where}: is_fisheye cameras are not supported")
        for k in ('k3', 'k4'):
            if float(meta.get(k, 0.0)) != 0.0:
                raise ValueError(f"{where}: a non-zero {k} is not supported (k1 k2 p1 p2 are)")
        cx = meta['cx'] * self.downsample if 'cx' in meta else w / 2
        cy = meta['cy'] * self.downsample if 'cy' in meta else h / 2
        dist = tuple(float(meta.get(k, 0.0)) for k in ('k1', 'k2', 'p1', 'p2'))
        self.camera = Camera('OPENCV', fx, fy, cx, cy, dist)
        self.K = self.camera.K()
        self.directions = get_ray_directions(h, w, self.K)   # the pinhole table until to(device) unprojects
        self.img_wh = (w, h)

    def read_meta(self, split):
        meta = self._meta()
        with_depth = any('depth_path' in f for f in meta['frames'])
        if with_depth and 'integer_depth_scale' not in meta:
            raise ValueError(f"{self.root_dir}/transforms.json: frames have depth_path but no integer_depth_scale")
        poses, imgs, depths = [], [], []
        for frame in meta['frames']:
            path = os.path.join(self.root_dir, f"{frame['file_path']}")
            if not os.path.exists(path):
                continue
            imgs.append(read_image(path, self.img_wh, keep_alpha=True))
            c2w = np.array(frame['transform_matrix'], dtype=np.float64)[:3, :4]
            c2w[:, 1:3] *= -1
            poses.append(c2w)
            if with_depth:
                depths.append(self._read_depth(frame, meta) if 'depth_path' in frame
                              else np.zeros(self.img_wh[0] * self.img_wh[1], np.float32))
        self.rays = stack_images(imgs)
        self.poses = stack_poses(poses)
        if with_depth:
            self.depths = torch.from_numpy(np.stack(depths)) if depths else torch.empty(0)

    def _read_depth(self, frame, meta):
        """[H*W] fp32 z-depth of one frame's depth image, nearest-neighbour resampled to ``img_wh``."""
        path = os.path.join(self.root_dir, frame['depth_path'])
        with Image.open(path) as im:
            if im.mode not in ('I;16', 'I;16B', 'I;16L', 'I', 'L'):
                raise ValueError(f"{path}: depth image mode {im.mode!r}; depth must be a single-channel integer image")
            if im.size != (int(meta['w']), int(meta['h'])):
                raise ValueError(f"{path}: depth image is {im.size[0]}x{im.size[1]}, transforms.json says "
                                 f"{meta['w']}x{meta['h']}")
            raw = np.asarray(im).astype(np.float64)
        (w, h), (W, H) = self.img_wh, im.size
        # nearest neighbour: output pixel centre (x + 0.5) W / w falls in source pixel floor of it
        xs = np.minimum(((np.arange(w) + 0.5) * W / w).astype(np.int64), W - 1)
        ys = np.minimum(((np.arange(h) + 0.5) * H / h).astype(np.int64), H - 1)
        return (raw[ys[:, None], xs[None, :]] * float(meta['integer_depth_scale'])).astype(np.float32).reshape(-1)
