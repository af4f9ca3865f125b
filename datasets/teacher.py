"""Teacher dataset: views of the reference's SHIPPED, TRAINED Lego model.

No NeRF dataset exists offline (SURVEY.md §8c), so "PSNR vs ref" is measured against a teacher: the only trained
artefact the reference ships — its mobile-demo Lego model (deployment/InstantNGP/taichi_ngp/compiled/*.bin: L=4 F=4
dense grid, 16-wide MLPs, occupancy bitfield), rebuilt git-ignored under oracle/_ref/lego_deployment from
tests/golden/ by ``__graft_entry__.build()``.  The teacher is loaded with ``modules.utils.load_deployment_model`` and rendered with the
CUDA path (``render(test_time=True)``, T_threshold 1e-2 as the demo uses, white background); the images then play
the role of datasets/nsvf.py's ``self.rays`` (train split) / per-view ``rgb`` (test split), with the Synthetic-NeRF
Lego intrinsics (datasets/nsvf.py:37-44) and cameras on the upper hemisphere at the shipped pose's radius (1.396).
"""
from __future__ import annotations

import os

import torch

from .ray_utils import get_rays
from .synthetic import SyntheticLego

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEACHER_FILES = ("hash_embedding", "sigma_weights", "rgb_weights", "density_bitfield")


def teacher_dir():
    d = os.environ.get("NGP_TEACHER_DIR", os.path.join(_ROOT, "oracle", "_ref", "lego_deployment"))
    return d if all(os.path.exists(os.path.join(d, n + ".bin")) for n in TEACHER_FILES) else None


def load_teacher(device):
    """The shipped Lego model as an ``NGP`` (deployment config, train.py:88-99), or None when it is not staged."""
    d = teacher_dir()
    if d is None:
        return None
    from modules.networks import NGP
    from modules.utils import load_deployment_model
    model = NGP(scale=0.5, pos_encoder_type='hash', levels=4, feature_per_level=4, base_res=32, max_res=128,
                log2_T=21, xyz_net_width=16, rgb_net_width=16, rgb_net_depth=1).to(device)
    load_deployment_model(model, d)
    return model.eval()


@torch.no_grad()
def render_views(model, directions, poses, T_threshold=1e-2, return_depth=False):
    """[n_views, H*W, 3] fp32 images of ``model`` (white background) for (3,4) camera-to-world ``poses``; with
    ``return_depth`` also [n_views, H*W] fp32 the render's expected z-depth sum_k w_k t_k."""
    from modules.rendering import render
    out, dep = [], []
    for pose in poses:
        rays_o, rays_d = get_rays(directions, pose)
        with torch.autocast('cuda', dtype=torch.float16):
            res = render(model, rays_o, rays_d, test_time=True, T_threshold=T_threshold, exp_step_factor=0.0)
        out.append(res['rgb'].float().clamp(0, 1))
        dep.append(res['depth'].float())
    return (torch.stack(out), torch.stack(dep)) if return_depth else torch.stack(out)


class TeacherLego(SyntheticLego):
    """``SyntheticLego`` geometry with target colours rendered from the shipped Lego model."""

    def __init__(self, n_images: int = 48, radius: float = 1.396, with_depth: bool = False, **kw):
        kw.pop('scene', None)
        super().__init__(n_images=n_images, radius=radius, scene='teacher', **kw)
        self.images = None            # [n_images, H*W, 3] once rendered (needs the GPU)
        self.with_depth = with_depth  # samples also carry 'depth', the teacher render's z-depth (DESIGN.md §6h)
        self.depths = None            # [n_images, H*W] once rendered, with_depth only

    def to(self, device):
        super().to(device)
        if self.images is not None:
            self.images = self.images.to(device)
        if self.depths is not None:
            self.depths = self.depths.to(device)
        return self

    def build_image_bank(self, teacher=None):
        if self.images is None:
            dev = self.poses.device
            teacher = teacher if teacher is not None else load_teacher(dev)
            if teacher is None:
                raise FileNotFoundError("teacher model not staged: run __graft_entry__.build(), "
                                        "or set NGP_TEACHER_DIR to a folder with the six .bin files")
            if self.with_depth:
                self.images, self.depths = render_views(teacher, self.directions, self.poses, return_depth=True)
            else:
                self.images = render_views(teacher, self.directions, self.poses)
        self.rays = self.images
        return self.rays

    def gather(self, img, pix):
        """The training sample of the rays (img[i], pix[i]), as ``dataset[idx]`` returns it for those indices."""
        if self.images is None:
            self.build_image_bank()
        sample = {'img_idxs': img, 'pix_idxs': pix, 'pose': self.poses[img], 'direction': self.directions[pix],
                  'rgb': self.images[img, pix]}
        if self.with_depth:
            sample['depth'] = self.depths[img, pix]
        return sample

    def __getitem__(self, idx):
        if self.images is None:
            self.build_image_bank()
        dev = self.poses.device
        if self.split.startswith('train'):
            img, pix = self._draw(idx, self.batch_size, dev)
            return self.gather(img, pix)
        sample = {'pose': self.poses[idx], 'img_idxs': idx, 'rgb': self.images[idx]}
        if self.with_depth:
            sample['depth'] = self.depths[idx]
        return sample
