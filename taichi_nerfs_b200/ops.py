"""Thin torch-tensor front ends of the C-ABI calls (no autograd here; see modules/).

Every function takes CUDA tensors, passes raw ``data_ptr()``s and the CURRENT torch stream to
libngp_b200 and returns/updates caller-visible tensors — the same contract the reference has
with Taichi ndarrays (contiguous tensors, shared CUDA context, async launches).
PyTorch is plumbing (allocation, streams); all arithmetic happens in the CUDA library.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import F16, F32, check, load


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.NgpError("libngp_b200 ops need CUDA tensors (there is no CPU fallback)")


def _tag(t):
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.float32:
        return F32
    raise TypeError(f"unsupported dtype {t.dtype}")


def _f32c(t):
    return t.contiguous() if t.dtype == torch.float32 else t.float().contiguous()


# ---- a1 ------------------------------------------------------------------------------------------
def ray_aabb_intersect(rays_o, rays_d, scale):
    _need_cuda(rays_o, rays_d)
    o, d = _f32c(rays_o), _f32c(rays_d)
    hits = torch.empty(o.shape[0], 2, device=o.device, dtype=torch.float32)
    check(load().ngp_ray_aabb_intersect(_ptr(o), _ptr(d), float(scale), _ptr(hits), o.shape[0], _stream()),
          "ray_aabb_intersect")
    return hits


# ---- a2 ------------------------------------------------------------------------------------------
def raymarching_train_count(rays_o, rays_d, hits_t, bitfield, noise, cascades, scale, exp_step_factor,
                            grid_size, max_samples, counter=None, rays_a=None):
    _need_cuda(rays_o, rays_d, hits_t, bitfield, noise)
    n = rays_o.shape[0]
    if counter is None:
        counter = torch.empty(2, device=rays_o.device, dtype=torch.int32)
    if rays_a is None:
        rays_a = torch.empty(n, 3, device=rays_o.device, dtype=torch.int32)
    check(load().ngp_raymarching_train_count(_ptr(rays_o), _ptr(rays_d), _ptr(hits_t), _ptr(bitfield), _ptr(noise),
                                             int(cascades), int(grid_size), float(scale), float(exp_step_factor),
                                             int(max_samples), _ptr(counter), _ptr(rays_a), n, _stream()),
          "raymarching_train_count")
    return counter, rays_a


def raymarching_train_write(rays_o, rays_d, hits_t, bitfield, noise, cascades, scale, exp_step_factor, grid_size,
                            counter, rays_a, xyzs, dirs, deltas, ts):
    n = rays_o.shape[0]
    cap = deltas.shape[0]
    check(load().ngp_raymarching_train_write(_ptr(rays_o), _ptr(rays_d), _ptr(hits_t), _ptr(bitfield), _ptr(noise),
                                             int(cascades), int(grid_size), float(scale), float(exp_step_factor),
                                             _ptr(counter), _ptr(rays_a), _ptr(xyzs), _ptr(dirs), _ptr(deltas),
                                             _ptr(ts), n, cap, _stream()),
          "raymarching_train_write")


def raymarching_frame(rays_o, rays_d, hits_t, bitfield, cascades, scale, exp_step_factor, grid_size, max_samples,
                      counter, rays_a, xyzs, dirs, deltas, ts, noise=None):
    """Single-pass march into capacity buffers; counter = [rows reserved, rays dropped] (caller zeroes it).
    noise=None: test-time semantics; noise tensor: training semantics (jittered start)."""
    n, cap = rays_o.shape[0], deltas.shape[0]
    check(load().ngp_raymarching_frame(_ptr(rays_o), _ptr(rays_d), _ptr(hits_t), _ptr(noise), _ptr(bitfield), int(cascades),
                                       int(grid_size), float(scale), float(exp_step_factor), int(max_samples),
                                       _ptr(counter), _ptr(rays_a), _ptr(xyzs), _ptr(dirs), _ptr(deltas), _ptr(ts),
                                       n, cap, _stream()), "raymarching_frame")


# ---- a3 ------------------------------------------------------------------------------------------
def raymarching_test(rays_o, rays_d, hits_t, alive_indices, bitfield, cascades, scale, exp_step_factor, grid_size,
                     max_samples, ray_indices, valid_mask, deltas, ts, samples_counter):
    _need_cuda(rays_o, rays_d, hits_t, alive_indices, bitfield)
    check(load().ngp_raymarching_test(_ptr(rays_o), _ptr(rays_d), _ptr(hits_t), _ptr(alive_indices), _ptr(bitfield),
                                      int(cascades), int(grid_size), float(scale), float(exp_step_factor),
                                      int(max_samples), _ptr(ray_indices), _ptr(valid_mask), _ptr(deltas), _ptr(ts),
                                      _ptr(samples_counter), alive_indices.shape[0], _stream()),
          "raymarching_test")


# ---- a4/a5 ---------------------------------------------------------------------------------------
def hash_encode_fwd(xyz, table, clayout, out_dim, aabb=None):
    """aabb = (xyz_min[3], xyz_max-xyz_min[3]) folds NGP.density's normalisation into the kernel."""
    _need_cuda(xyz, table)
    n = xyz.shape[0]
    out = torch.empty(n, out_dim, device=xyz.device, dtype=table.dtype)
    if aabb is None:
        check(load().ngp_hash_encode_fwd(_ptr(xyz), _ptr(table), C.byref(clayout), _ptr(out), _tag(table), n,
                                         _stream()), "hash_encode_fwd")
    else:
        a6 = (C.c_float * 6)(*[float(v) for v in aabb])
        check(load().ngp_hash_encode_fwd_dyn(_ptr(xyz), _ptr(table), C.byref(clayout), _ptr(out), _tag(table), n,
                                             None, a6, _stream()), "hash_encode_fwd_dyn")
    return out


def hash_encode_bwd(xyz, dout, clayout, grad_table):
    _need_cuda(xyz, dout, grad_table)
    check(load().ngp_hash_encode_bwd(_ptr(xyz), _ptr(dout), _tag(dout), C.byref(clayout), _ptr(grad_table),
                                     xyz.shape[0], _stream()),
          "hash_encode_bwd")
    return grad_table


def hash_encode_bwd_input(xyz, table, dout, clayout):
    _need_cuda(xyz, table, dout)
    dx = torch.empty(xyz.shape[0], 3, device=xyz.device, dtype=torch.float32)
    check(load().ngp_hash_encode_bwd_input(_ptr(xyz), _ptr(table), _ptr(dout), _tag(table), C.byref(clayout),
                                           _ptr(dx), xyz.shape[0], _stream()),
          "hash_encode_bwd_input")
    return dx


# ---- tri-plane encoder -----------------------------------------------------------------------------
def triplane_encode_fwd(xyz, table, clayout, aabb=None, out=None):
    """xyz [n,3] fp32 in [0,1] (or world positions with aabb = (xyz_min[3], xyz_max-xyz_min[3]), normalised in the
    kernel) -> fp32 [n, L*F] in the reference's feature-major column order."""
    _need_cuda(xyz, table, out)
    if xyz.dtype != torch.float32 or table.dtype != torch.float32:
        raise TypeError("triplane_encode_fwd: positions and the plane table must be fp32")
    n = xyz.shape[0]
    if out is None:
        out = torch.empty(n, clayout.n_levels * clayout.feat_dim, device=xyz.device, dtype=torch.float32)
    a6 = None if aabb is None else (C.c_float * 6)(*[float(v) for v in aabb])
    check(load().ngp_triplane_encode_fwd(_ptr(xyz), _ptr(table), C.byref(clayout), _ptr(out), n, a6, _stream()),
          "triplane_encode_fwd")
    return out


def triplane_encode_bwd(xyz, table, dout, clayout, grad_table):
    """grad_table (fp32 [P]) += dL/dtable for dout fp32 [n, L*F]; xyz in [0,1]."""
    _need_cuda(xyz, table, dout, grad_table)
    if dout.dtype != torch.float32 or grad_table.dtype != torch.float32:
        raise TypeError("triplane_encode_bwd: dout and grad_table must be fp32")
    check(load().ngp_triplane_encode_bwd(_ptr(xyz), _ptr(table), _ptr(dout), C.byref(clayout), _ptr(grad_table),
                                         xyz.shape[0], _stream()), "triplane_encode_bwd")
    return grad_table


# ---- a6 ------------------------------------------------------------------------------------------
def dir_encode(dirs):
    _need_cuda(dirs)
    d = _f32c(dirs)
    out = torch.empty(d.shape[0], 16, device=d.device, dtype=torch.float32)
    check(load().ngp_dir_encode(_ptr(d), _ptr(out), d.shape[0], _stream()), "dir_encode")
    return out


# ---- a8 ------------------------------------------------------------------------------------------
def composite_train_fwd(sigmas, rgbs, deltas, ts, rays_a, T_threshold):
    _need_cuda(sigmas, rgbs, deltas, ts, rays_a)
    n, S = rays_a.shape[0], sigmas.shape[0]
    dev = rays_a.device
    total = torch.empty(n, device=dev, dtype=torch.int32)
    opacity = torch.empty(n, device=dev, dtype=torch.float32)
    depth = torch.empty(n, device=dev, dtype=torch.float32)
    rgb = torch.empty(n, 3, device=dev, dtype=torch.float32)
    ws = torch.empty(S, device=dev, dtype=torch.float32)
    check(load().ngp_composite_train_fwd(_ptr(sigmas), _ptr(rgbs), _tag(rgbs), _ptr(deltas), _ptr(ts), _ptr(rays_a),
                                         float(T_threshold), _ptr(total), _ptr(opacity), _ptr(depth), _ptr(rgb),
                                         _ptr(ws), n, S, _stream()),
          "composite_train_fwd")
    return total, opacity, depth, rgb, ws


def composite_train_bwd(dL_dopacity, dL_ddepth, dL_drgb, dL_dws, sigmas, rgbs, deltas, ts, rays_a, T_threshold):
    n, S = rays_a.shape[0], sigmas.shape[0]
    dsig = torch.zeros(S, device=sigmas.device, dtype=torch.float32)
    drgbs = torch.zeros(S, 3, device=sigmas.device, dtype=rgbs.dtype)
    check(load().ngp_composite_train_bwd(_ptr(dL_dopacity), _ptr(dL_ddepth), _ptr(dL_drgb), _ptr(dL_dws),
                                         _ptr(sigmas), _ptr(rgbs), _tag(rgbs), _ptr(deltas), _ptr(ts), _ptr(rays_a),
                                         None, None, None, float(T_threshold), _ptr(dsig), _ptr(drgbs), n, S,
                                         _stream()),
          "composite_train_bwd")
    return dsig, drgbs


# ---- a9 ------------------------------------------------------------------------------------------
def composite_test(sigmas, rgbs, deltas, ts, pack_info, alive_indices, T_threshold, opacity, depth, rgb):
    _need_cuda(sigmas, rgbs, deltas, ts, pack_info, alive_indices, opacity, depth, rgb)
    check(load().ngp_composite_test(_ptr(sigmas), _ptr(rgbs), _tag(rgbs), _ptr(deltas), _ptr(ts), _ptr(pack_info),
                                    _ptr(alive_indices), float(T_threshold), _ptr(opacity), _ptr(depth), _ptr(rgb),
                                    alive_indices.shape[0], _stream()),
          "composite_test")


# ---- distortion loss ---------------------------------------------------------------------------------
def distortion_fwd(ws, deltas, ts, rays_a):
    _need_cuda(ws, deltas, ts, rays_a)
    loss = torch.zeros(rays_a.shape[0], device=ws.device, dtype=torch.float32)
    check(load().ngp_distortion_fwd(_ptr(ws), _ptr(deltas), _ptr(ts), _ptr(rays_a), _ptr(loss), rays_a.shape[0],
                                    ws.shape[0], _stream()), "distortion_fwd")
    return loss


def distortion_bwd(dL_dloss, ws, deltas, ts, rays_a):
    out = torch.zeros_like(ws)
    check(load().ngp_distortion_bwd(_ptr(dL_dloss), _ptr(ws), _ptr(deltas), _ptr(ts), _ptr(rays_a), _ptr(out),
                                    rays_a.shape[0], ws.shape[0], _stream()), "distortion_bwd")
    return out


# ---- occupancy grid helpers ------------------------------------------------------------------------
def packbits(density_grid, threshold, bitfield, mean_dev=None):
    """bit i of byte n = grid[8n+i] > thr, thr = threshold or min(*mean_dev, threshold) read on the device."""
    _need_cuda(density_grid, bitfield)
    if mean_dev is None:
        check(load().ngp_packbits(_ptr(density_grid), float(threshold), _ptr(bitfield), bitfield.shape[0], _stream()),
              "packbits")
    else:
        m = mean_dev.float().contiguous()
        check(load().ngp_packbits_dev(_ptr(density_grid), _ptr(m), float(threshold), _ptr(bitfield),
                                      bitfield.shape[0], _stream()), "packbits_dev")


# ---- f1: fused occupancy-grid update ------------------------------------------------------------------
def grid_workspace(cascades, grid_size, device):
    n = int(load().ngp_grid_workspace_bytes(int(cascades), int(grid_size)))
    return torch.empty(n, device=device, dtype=torch.uint8)


def grid_sample_cells(density_grid, scale, density_threshold, warmup, M, seed, step, workspace):
    """Cells to evaluate + their jittered world positions (networks.py:168-209, 263-271) -> (cell_idx [C*slots] i32,
    xyz [C*slots, 3] f32); slots = grid_size^3 (warm-up) or 2*M."""
    _need_cuda(density_grid, workspace)
    cascades, cells = density_grid.shape
    G = round(cells ** (1 / 3))
    slots = cells if warmup else 2 * int(M)
    cell_idx = torch.empty(cascades * slots, device=density_grid.device, dtype=torch.int32)
    xyz = torch.empty(cascades * slots, 3, device=density_grid.device, dtype=torch.float32)
    check(load().ngp_grid_sample_cells(_ptr(density_grid), cascades, G, float(scale), float(density_threshold),
                                       0 if warmup else 1, int(M), int(seed), int(step) & 0xFFFFFFFF, _ptr(workspace),
                                       _ptr(cell_idx), _ptr(xyz), _stream()), "grid_sample_cells")
    return cell_idx, xyz


def grid_update(density_grid, cell_idx, densities, density_threshold, decay, workspace, mean_out, bitfield,
                count_grid=None):
    """Scatter-max + EMA-max + mean of the positive cells + packbits (networks.py:272-290), in place, no host sync."""
    _need_cuda(density_grid, cell_idx, densities, workspace, mean_out, bitfield)
    cascades, cells = density_grid.shape
    G = round(cells ** (1 / 3))
    check(load().ngp_grid_update(_ptr(density_grid), _ptr(cell_idx), _ptr(densities), cell_idx.numel() // cascades,
                                 cascades, G, _ptr(count_grid), float(decay), float(density_threshold), _ptr(workspace),
                                 _ptr(mean_out), _ptr(bitfield), _stream()), "grid_update")


def sample_ray_batch(image_bank, poses, directions, n_rays, *, img_idxs=None, pix_idxs=None, fixed_img=-1, seed=0,
                     step=0, step_dev=None, with_noise=True, return_indices=False, out=None):
    """One launch for BaseDataset.__getitem__ + get_rays + the marching jitter (include/ngp_b200.h,
    ngp_sample_ray_batch).  ``out`` = optional dict of preallocated rays_o / rays_d / rgb / noise (graph capture)."""
    _need_cuda(poses, directions)
    dev = poses.device
    bank = None if image_bank is None else _f32c(image_bank)
    poses, directions = _f32c(poses), _f32c(directions)
    n_img, n_pix = poses.shape[0], directions.shape[0]
    if bank is not None and tuple(bank.shape[:2]) != (n_img, n_pix):
        raise ValueError(f"image bank {tuple(bank.shape)} does not match {n_img} poses x {n_pix} pixels")
    out = {} if out is None else out
    f = lambda k, *s: out[k] if k in out else torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    rays_o, rays_d = f("rays_o", n_rays, 3), f("rays_d", n_rays, 3)
    rgb = None if bank is None else f("rgb", n_rays, 3)
    noise = f("noise", n_rays) if with_noise else None
    ii = pi = None
    if return_indices:
        ii = torch.empty(n_rays, device=dev, dtype=torch.int64)
        pi = torch.empty(n_rays, device=dev, dtype=torch.int64)
    img_in = None if img_idxs is None else img_idxs.to(torch.int64).contiguous()
    pix_in = None if pix_idxs is None else pix_idxs.to(torch.int64).contiguous()
    check(load().ngp_sample_ray_batch(_ptr(bank), 0 if bank is None else bank.shape[2], _ptr(poses), _ptr(directions),
                                      n_img, n_pix, _ptr(img_in), _ptr(pix_in), int(fixed_img), int(seed),
                                      _ptr(step_dev), int(step), _ptr(rays_o), _ptr(rays_d), _ptr(rgb), _ptr(noise),
                                      _ptr(ii), _ptr(pi), n_rays, _stream()), "sample_ray_batch")
    res = {"rays_o": rays_o, "rays_d": rays_d, "rgb": rgb, "noise": noise}
    if return_indices:
        res["img_idxs"], res["pix_idxs"] = ii, pi
    return res


def morton3d(coords):
    _need_cuda(coords)
    c = coords.contiguous()
    out = torch.empty(c.shape[0], device=c.device, dtype=torch.int32)
    check(load().ngp_morton3d(_ptr(c), _ptr(out), c.shape[0], _stream()), "morton3d")
    return out


def morton3d_invert(indices):
    _need_cuda(indices)
    i = indices.contiguous()
    out = torch.empty(i.shape[0], 3, device=i.device, dtype=torch.int32)
    check(load().ngp_morton3d_invert(_ptr(i), _ptr(out), i.shape[0], _stream()), "morton3d_invert")
    return out


# ---- a12 -----------------------------------------------------------------------------------------
def adam_step(param, grad, exp_avg, exp_avg_sq, lr, step, beta1=0.9, beta2=0.999, eps=1e-15, inv_scale=1.0,
              param_f16=None, found_inf=None, zero_grad=False):
    _need_cuda(param, grad, exp_avg, exp_avg_sq)
    check(load().ngp_adam_step(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(param_f16),
                               _ptr(found_inf), float(lr), float(beta1), float(beta2), float(eps), float(inv_scale),
                               int(step), int(bool(zero_grad)), param.numel(), _stream()),
          "adam_step")


def check_finite(grad, found_inf):
    _need_cuda(grad, found_inf)
    check(load().ngp_check_finite(_ptr(grad), grad.numel(), _ptr(found_inf), _stream()), "check_finite")


# ---- a7 ------------------------------------------------------------------------------------------
def _mlp_weights(ws):
    """ws: 5 fp32 CUDA tensors shaped like the nn.Linear weights [64,32],[16,64],[64,32],[64,64],[3,64]."""
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    keep = []
    for w, s in zip(ws, shapes):
        if tuple(w.shape) != s:
            raise ValueError(f"fused MLP expects weight shape {s}, got {tuple(w.shape)}")
        keep.append(w.detach().float().contiguous())
    return _lib.MlpWeights(*[k.data_ptr() for k in keep]), keep


def mlp_fwd(emb, dirs, ws, with_save=False):
    """emb [n,32] fp16/fp32, dirs [n,3] fp32 (un-normalised) -> sigmas [n] fp32, rgbs [n,3] fp16
    [, save: the activations the backward restarts from (ngp_mlp_save_bytes(n) bytes)]."""
    _need_cuda(emb, dirs)
    n = emb.shape[0]
    emb = emb.contiguous()
    d = _f32c(dirs)
    st, keep = _mlp_weights(ws)
    sig = torch.empty(n, device=emb.device, dtype=torch.float32)
    rgb = torch.empty(n, 3, device=emb.device, dtype=torch.float16)
    save = None
    if with_save:
        save = torch.empty(max(int(load().ngp_mlp_save_bytes(n)), 16), device=emb.device, dtype=torch.uint8)
    check(load().ngp_mlp_fwd(_ptr(emb), _tag(emb), _ptr(d), C.byref(st), _ptr(sig), _ptr(rgb), _ptr(save), n, _stream()),
          "mlp_fwd")
    return (sig, rgb, save) if with_save else (sig, rgb)


def mlp_bwd(emb, dirs, ws, dsigmas, drgbs, save=None):
    """-> demb [n,32] (emb dtype), grad_w fp32 [9408] in the order w1|w2|w3|w4|w5.  ``save`` = the buffer returned
    by mlp_fwd(..., with_save=True) on the same inputs (None: everything is recomputed from emb / dirs)."""
    _need_cuda(emb, dirs, dsigmas, drgbs)
    n = emb.shape[0]
    emb = emb.contiguous()
    d = _f32c(dirs)
    st, keep = _mlp_weights(ws)
    demb = torch.empty(n, 32, device=emb.device, dtype=emb.dtype)
    gw = torch.zeros(9408, device=emb.device, dtype=torch.float32)
    check(load().ngp_mlp_bwd(_ptr(emb), _tag(emb), _ptr(d), C.byref(st), _ptr(save), _ptr(_f32c(dsigmas)),
                             _ptr(drgbs.to(torch.float16).contiguous()), _ptr(demb), _ptr(gw), n, _stream()),
          "mlp_bwd")
    return demb, gw
