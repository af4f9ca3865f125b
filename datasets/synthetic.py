"""Synthetic "Lego-shape" dataset: the geometry of the reference's Synthetic-NeRF/NSVF Lego setup
(800x800 pinhole, fx=fy=1111.111 — datasets/nsvf.py:37-44; cameras on the upper hemisphere looking at
the origin, scene in [-0.5,0.5]^3) with random target colours.  No image files are available offline,
so this stands in for datasets/{nsvf,nerf}.py on the benchmark path (BASELINE.md §4).

Follows the BaseDataset protocol of the reference (datasets/base.py:6-61): ``dataset[i]`` in a train
split returns {'img_idxs','pix_idxs','pose','direction','rgb'} for ``batch_size`` random rays.
"""
from __future__ import annotations

import math

import torch

from .ray_utils import get_ray_directions


def hemisphere_poses(n_poses: int, radius: float = 1.4, seed: int = 23) -> torch.Tensor:
    """(n,3,4) camera-to-world matrices, columns = [right, down, front, position]."""
    g = torch.Generator().manual_seed(seed)
    theta = torch.rand(n_poses, generator=g) * 2 * math.pi
    phi = torch.acos(torch.rand(n_poses, generator=g) * 0.9 + 0.05)  # elevation away from the horizon/pole
    pos = torch.stack([torch.sin(phi) * torch.cos(theta), torch.sin(phi) * torch.sin(theta), torch.cos(phi)], -1) * radius
    front = -pos / pos.norm(dim=-1, keepdim=True)
    up = torch.tensor([0.0, 0.0, 1.0]).expand_as(front)
    right = torch.cross(front, up, dim=-1)
    right = right / right.norm(dim=-1, keepdim=True)
    down = torch.cross(front, right, dim=-1)
    return torch.stack([right, down, front, pos], dim=-1).float()


def analytic_scene(x):
    """Closed-form teacher radiance field inside [-0.5,0.5]^3: three soft blobs and a box frame.
    x: (..., 3) -> (sigma (...), rgb (..., 3))."""
    centers = x.new_tensor([[0.15, 0.0, -0.1], [-0.2, 0.15, 0.05], [0.0, -0.2, 0.2]])
    radii = x.new_tensor([0.18, 0.14, 0.10])
    colors = x.new_tensor([[0.9, 0.75, 0.1], [0.1, 0.5, 0.9], [0.85, 0.2, 0.2]])
    d2 = ((x[..., None, :] - centers) ** 2).sum(-1)                       # (..., 3)
    dens = 60.0 * torch.sigmoid((radii ** 2 - d2) * 400.0)                 # soft spheres
    sigma = dens.sum(-1)
    rgb = (dens[..., None] * colors).sum(-2) / (sigma[..., None] + 1e-6)
    return sigma, rgb.clamp(0, 1)


@torch.no_grad()
def render_teacher(rays_o, rays_d, n_samples: int = 192, scale: float = 0.5, return_depth: bool = False):
    """Quadrature volume rendering of `analytic_scene` on a white background (synthetic-scene convention).  With
    ``return_depth`` also the quadrature's expected depth sum_k w_k t_k (no background term): z-depth, since ``rays_d``
    is the unnormalised camera-frame direction (u', v', 1) rotated to the world."""
    inv = 1.0 / rays_d
    t0 = ((-scale - rays_o) * inv)
    t1 = ((scale - rays_o) * inv)
    near = torch.minimum(t0, t1).amax(-1).clamp_min(0.01)
    far = torch.maximum(t0, t1).amin(-1)
    hit = far > near
    u = (torch.arange(n_samples, device=rays_o.device) + 0.5) / n_samples
    t = near[:, None] + (far - near).clamp_min(0)[:, None] * u
    dt = ((far - near).clamp_min(0) / n_samples)[:, None]
    x = rays_o[:, None, :] + t[..., None] * rays_d[:, None, :]
    sigma, rgb = analytic_scene(x)
    alpha = 1 - torch.exp(-sigma * dt)
    T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], 1), 1)[:, :-1]
    w = alpha * T * hit[:, None]
    out = (w[..., None] * rgb).sum(1) + (1 - w.sum(1))[:, None]
    return (out, (w * t).sum(1)) if return_depth else out


class SyntheticLego:
    def __init__(self, n_images: int = 100, img_wh=(800, 800), focal: float = 1111.111, radius: float = 1.4,
                 split: str = 'train', batch_size: int = 8192, seed: int = 23, with_rgb: bool = True,
                 scene: str = 'random', root_dir: str = '', downsample: float = 1.0, with_depth: bool = False, **_):
        w, h = int(img_wh[0] * downsample), int(img_wh[1] * downsample)
        focal = focal * downsample
        if split != 'train' and not split.startswith('train'):
            seed = seed + 1000  # held-out poses
        self.scene = scene
        self.img_wh = (w, h)
        self.split = split
        self.batch_size = batch_size
        self.ray_sampling_strategy = 'all_images'
        self.K = torch.tensor([[focal, 0, w / 2], [0, focal, h / 2], [0, 0, 1]], dtype=torch.float32)
        self.directions = get_ray_directions(h, w, self.K)
        self.poses = hemisphere_poses(n_images, radius, seed)
        self._gen = None
        self.rays = None
        self._seed = seed
        self.with_rgb = with_rgb
        # with_depth (the analytic scene): samples also carry 'depth', the teacher's expected z-depth (DESIGN.md §6h)
        if with_depth and scene != 'analytic':
            raise ValueError("SyntheticLego: with_depth needs scene='analytic' (the random scene has no geometry)")
        self.with_depth = with_depth

    def __len__(self):
        return len(self.poses)

    def to(self, device):
        self.K = self.K.to(device)
        self.directions = self.directions.to(device)
        self.poses = self.poses.to(device)
        if self.rays is not None:
            self.rays = self.rays.to(device)
        return self

    def build_image_bank(self):
        """``self.rays`` [n_images, H*W, 3]: every training pixel resident, as the reference's datasets keep them
        (datasets/nsvf.py / colmap.py ``self.rays``; moved to the GPU by BaseDataset.to, base.py:26-31).  Needed by
        the on-device batch sampler (ngp_sample_ray_batch / StaticTrainStep.attach_ray_source)."""
        dev = self.poses.device
        n_pix = self.img_wh[0] * self.img_wh[1]
        if self.scene == 'analytic':
            from .ray_utils import get_rays
            imgs = []
            for pose in self.poses:
                o, d = get_rays(self.directions, pose)
                imgs.append(torch.cat([render_teacher(o[i:i + 65536], d[i:i + 65536]) for i in range(0, n_pix, 65536)]))
            self.rays = torch.stack(imgs)
        else:
            g = torch.Generator(device=dev).manual_seed(self._seed + 7)
            self.rays = torch.rand(len(self.poses), n_pix, 3, device=dev, generator=g)
        return self.rays

    def _draw(self, idx, n, dev):
        """(image index, pixel index) of a training batch: datasets/base.py:34-52 ('all_images': every ray from a
        random image; 'same_image': all rays of the batch from image ``idx``)."""
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(self._seed)
        if self.ray_sampling_strategy == 'same_image':
            img = torch.full((n,), int(idx) % len(self.poses), device=dev, dtype=torch.long)
        elif self.ray_sampling_strategy == 'all_images':
            img = torch.randint(0, len(self.poses), (n,), device=dev, generator=self._gen)
        else:
            raise ValueError(f"unknown ray_sampling_strategy {self.ray_sampling_strategy!r}")
        pix = torch.randint(0, self.img_wh[0] * self.img_wh[1], (n,), device=dev, generator=self._gen)
        return img, pix

    def gather(self, img, pix):
        """The training sample of the rays (img[i], pix[i]), as ``dataset[idx]`` returns it for those indices.  The
        random scene's colours are not a function of the pixel: they are drawn from the dataset's generator."""
        sample = {'img_idxs': img, 'pix_idxs': pix, 'pose': self.poses[img], 'direction': self.directions[pix]}
        if self.with_rgb:
            if self.scene == 'analytic':
                from .ray_utils import get_rays
                o, d = get_rays(sample['direction'], sample['pose'])
                if self.with_depth:
                    sample['rgb'], sample['depth'] = render_teacher(o, d, return_depth=True)
                else:
                    sample['rgb'] = render_teacher(o, d)
            else:
                dev = self.poses.device
                if self._gen is None or self._gen.device != dev:
                    self._gen = torch.Generator(device=dev).manual_seed(self._seed)
                sample['rgb'] = torch.rand(pix.shape[0], 3, device=dev, generator=self._gen)
        return sample

    def __getitem__(self, idx):
        dev = self.poses.device
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(self._seed)
        n = self.batch_size
        if self.split.startswith('train'):
            img, pix = self._draw(idx, n, dev)
            return self.gather(img, pix)
        sample = {'pose': self.poses[idx], 'img_idxs': idx}
        if self.scene == 'analytic':
            from .ray_utils import get_rays
            o, d = get_rays(self.directions, self.poses[idx])
            parts = [render_teacher(o[i:i + 65536], d[i:i + 65536], return_depth=self.with_depth)
                     for i in range(0, o.shape[0], 65536)]
            if self.with_depth:
                sample['rgb'], sample['depth'] = (torch.cat(p) for p in zip(*parts))
            else:
                sample['rgb'] = torch.cat(parts)
        return sample
