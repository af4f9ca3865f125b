"""Render orchestration — mirrors modules/rendering.py of the reference: render() :12-57,
test-time loop :61-158, training path :161-228.  Same signatures and result dictionaries."""
from __future__ import annotations

import torch

from .intersection import ray_aabb_intersection
from .ray_march import raymarching_test, raymarching_train
from .volume_render_test import composite_test

MAX_SAMPLES = 1024
NEAR_DISTANCE = 0.01


def render(model, rays_o, rays_d, test_time=False, exp_step_factor=0, T_threshold=1e-4,
           max_samples=MAX_SAMPLES, bg_rgb=None, position_grad=False, exposure=None):
    """AABB test, then the train or test rendering path.  Returns the result dict of the
    reference (train: rgb, depth, opacity, ws, deltas, ts, rays_a, rm_samples, vr_samples;
    test: rgb, depth, opacity, total_samples).  ``bg_rgb`` [N, 3] (training path only, --random_bg): each ray's own
    background colour in place of the fixed white / black one.  ``position_grad`` (training path only, camera
    extrinsics refinement, DESIGN.md §6i): the sample positions require grad and are returned as results['xyzs'], whose
    .grad the backward fills.  ``exposure`` (training path only, per-image exposure compensation, DESIGN.md §6k): a
    function (rgbs, rays_a) -> rgbs' that the network's sample colours pass through before compositing."""
    rays_o = rays_o.contiguous()
    rays_d = rays_d.contiguous()
    hits_t = ray_aabb_intersection(rays_o, rays_d, model.scale)
    if test_time:
        if getattr(model, '_fusable', None) is not None and rays_o.is_cuda:
            # same result as the incremental loop below, without its per-iteration host syncs
            from taichi_nerfs_b200.render_frame import render_frame, render_frame_compact
            if model._fusable(rays_o):
                # stock model: one CUDA graph per frame, live rays compacted between rounds (early termination)
                return render_frame_compact(model, rays_o, rays_d, exp_step_factor, T_threshold, max_samples)
            return render_frame(model, rays_o, rays_d, exp_step_factor, T_threshold, max_samples)
        return _render_rays_test(model, rays_o, rays_d, hits_t, exp_step_factor, T_threshold, max_samples)
    return _render_rays_train(model, rays_o, rays_d, hits_t, exp_step_factor, T_threshold, bg_rgb, position_grad,
                              exposure)


def _background(exp_step_factor, device):
    # synthetic scenes composite onto white, real scenes onto black (rendering.py:152-156, 219-224)
    return torch.ones(3, device=device) if exp_step_factor == 0 else torch.zeros(3, device=device)


@torch.no_grad()
def _render_rays_test(model, rays_o, rays_d, hits_t, exp_step_factor=0, T_threshold=1e-4,
                      max_samples=MAX_SAMPLES):
    n_rays = len(rays_o)
    device = rays_o.device
    opacity = torch.zeros(n_rays, device=device)
    depth = torch.zeros(n_rays, device=device)
    rgb = torch.zeros(n_rays, 3, device=device)

    samples = 0
    total_samples = 0
    alive = torch.arange(n_rays, device=device)
    min_samples = 1 if exp_step_factor == 0 else 4  # rendering.py:94

    while samples < max_samples:
        n_alive = len(alive)
        if n_alive == 0:
            break
        step = max(min(n_rays // n_alive, 64), min_samples)  # rendering.py:102
        samples += step
        pack_info, ray_indices, deltas, ts = raymarching_test(
            rays_o, rays_d, hits_t, alive, model.density_bitfield, model.cascades, model.scale,
            exp_step_factor, model.grid_size, step)
        if ray_indices.shape[0] == 0:
            break
        o = rays_o[ray_indices, :3]
        d = rays_d[ray_indices, :3]
        xyzs = o + ts[:, None] * d
        sigmas, rgbs = model(xyzs, d)
        composite_test(sigmas, rgbs, deltas, ts, pack_info, alive, T_threshold, opacity, depth, rgb)
        alive = alive[alive >= 0]
        total_samples += pack_info[:, 1].sum()

    results = {'opacity': opacity, 'depth': depth, 'rgb': rgb, 'total_samples': total_samples}
    results['rgb'] += _background(exp_step_factor, device) * (1 - opacity)[:, None]
    return results


def _render_rays_train(model, rays_o, rays_d, hits_t, exp_step_factor=0, T_threshold=1e-4, bg_rgb=None,
                       position_grad=False, exposure=None):
    results = {}
    (rays_a, xyzs, dirs, results['deltas'], results['ts'], results['rm_samples']) = raymarching_train(
        rays_o, rays_d, hits_t, model.density_bitfield, model.cascades, model.scale, exp_step_factor,
        model.grid_size, MAX_SAMPLES)
    if position_grad:
        results['xyzs'] = xyzs.requires_grad_(True)

    sigmas, rgbs = model(xyzs, dirs)
    if exposure is not None:
        rgbs = exposure(rgbs, rays_a)

    (results['vr_samples'], results['opacity'], results['depth'], results['rgb'], results['ws']) = \
        model.render_func(sigmas, rgbs, results['deltas'], results['ts'], rays_a, T_threshold)
    results['rays_a'] = rays_a

    bg = _background(exp_step_factor, rays_o.device) if bg_rgb is None else bg_rgb
    results['rgb'] = results['rgb'] + bg * (1 - results['opacity'])[:, None]
    return results
