"""Thin torch-tensor front ends of the C-ABI calls (no autograd here; see modules/).

Every function takes CUDA tensors, passes raw ``data_ptr()``s and the CURRENT torch stream to
libngp_b200 and returns/updates caller-visible tensors — the same contract the reference has
with Taichi ndarrays (contiguous tensors, shared CUDA context, async launches).
PyTorch is plumbing (allocation, streams); all arithmetic happens in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
import math

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
    """dL/dx [n, 3] fp32 of positions xyz in [0,1]; any feature width (the fixed-count entry takes F = 2 only, the
    device-counted one every width, with the same values at F = 2)."""
    return hash_encode_bwd_input_dyn(xyz, table, dout, clayout)


def hash_encode_bwd_input_dyn(xyz, table, dout, clayout, n_dev=None, aabb=None, out=None):
    """dL/dx [n, 3] fp32 over rows [0, min(n, n_dev[0])) (n_dev: int32 [1] device count, None: all n rows).  aabb =
    (xyz_min[3], xyz_max-xyz_min[3]): xyz are world positions and dx the world gradient (DESIGN.md §6i)."""
    _need_cuda(xyz, table, dout, n_dev, out)
    dx = torch.empty(xyz.shape[0], 3, device=xyz.device, dtype=torch.float32) if out is None else out
    a6 = None if aabb is None else (C.c_float * 6)(*[float(v) for v in aabb])
    check(load().ngp_hash_encode_bwd_input_dyn(_ptr(xyz), _ptr(table), _ptr(dout), _tag(table), C.byref(clayout),
                                               _ptr(dx), xyz.shape[0], _ptr(n_dev), a6, _stream()),
          "hash_encode_bwd_input_dyn")
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


# ---- voxel grid (--model_name svox) ------------------------------------------------------------------
VOXEL_BWD_WARP, VOXEL_BWD_THREAD = 0, 1     # NGP_VOXEL_BWD_* of include/ngp_b200.h


def _voxel_inputs(xyz, *fields):
    _need_cuda(xyz, *fields)
    for t in (xyz,) + fields:
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous()):
            raise TypeError("voxel ops take contiguous fp32 tensors")


def voxel_fwd(xyz, dirs, sh, density, clayout):
    """World positions xyz [n,3], directions dirs [n,3] (normalised in the kernel), fields sh [G,G,G,3D] and density
    [G,G,G,1] -> sigma [n], rgb [n,3], fp32.  dirs = None: density-only mode, returns sigma alone."""
    _voxel_inputs(xyz, dirs, sh, density)
    n = xyz.shape[0]
    sigma = torch.empty(n, device=xyz.device, dtype=torch.float32)
    rgb = None if dirs is None else torch.empty(n, 3, device=xyz.device, dtype=torch.float32)
    check(load().ngp_voxel_fwd(_ptr(xyz), _ptr(dirs), _ptr(sh), _ptr(density), C.byref(clayout), _ptr(sigma),
                               _ptr(rgb), n, _stream()), "voxel_fwd")
    return sigma if dirs is None else (sigma, rgb)


def voxel_bwd(xyz, dirs, sigma, rgb, dsigma, drgb, clayout, dsh, ddensity, found_inf=None, mapping=VOXEL_BWD_WARP):
    """dsh (fp32, sh-field sized) += dL/dsh and ddensity (fp32, density-field sized) += dL/ddensity, from the forward's
    outputs sigma / rgb and their gradients.  found_inf (int32 [1], optional) is raised on a non-finite gradient."""
    _voxel_inputs(xyz, dirs, sigma, rgb, dsigma, drgb, dsh, ddensity)
    check(load().ngp_voxel_bwd(_ptr(xyz), _ptr(dirs), _ptr(sigma), _ptr(rgb), _ptr(dsigma), _ptr(drgb),
                               C.byref(clayout), _ptr(dsh), _ptr(ddensity), xyz.shape[0], _ptr(found_inf),
                               int(mapping), _stream()), "voxel_bwd")


def voxel_bwd_dyn(xyz, dirs, sigma, rgb, dsigma, drgb, clayout, dsh, ddensity, n_dev=None, found_inf=None):
    """voxel_bwd (warp mapping) over rows [0, min(n, max(n_dev[0], 0))) with the count n_dev (int32 [1]) read on the
    device; n_dev None: all n rows."""
    _voxel_inputs(xyz, dirs, sigma, rgb, dsigma, drgb, dsh, ddensity)
    check(load().ngp_voxel_bwd_dyn(_ptr(xyz), _ptr(dirs), _ptr(sigma), _ptr(rgb), _ptr(dsigma), _ptr(drgb),
                                   C.byref(clayout), _ptr(dsh), _ptr(ddensity), xyz.shape[0], _ptr(n_dev),
                                   _ptr(found_inf), _stream()), "voxel_bwd_dyn")


def voxel_reg(sh, density, clayout, block, weights, dsh, ddensity, loss_scale=1.0, scale_dev=None, loss=None):
    """Total-variation and sparsity regularisers over the node block ``block`` = (lo_x, lo_y, lo_z, hi_x, hi_y, hi_z)
    (``layout.voxel_reg_block``): dsh += scale * dL/dsh and ddensity += scale * dL/ddensity for
    L = w_tv_sigma L_tv_sigma + w_tv_sh L_tv_sh + w_sparsity L_sparsity, ``weights`` = (w_tv_sigma, w_tv_sh,
    w_sparsity).  scale = scale_dev[0] (fp32 device tensor) when given, else loss_scale.  loss (fp32 [1], optional)
    accumulates the unscaled L.  All three weights 0: nothing is launched."""
    _voxel_inputs(sh, density, dsh, ddensity, scale_dev, loss)
    w_tv_sigma, w_tv_sh, w_sparsity = (float(w) for w in weights)
    b6 = (C.c_int32 * 6)(*[int(v) for v in block])
    check(load().ngp_voxel_reg(_ptr(sh), _ptr(density), C.byref(clayout), b6, w_tv_sigma, w_tv_sh, w_sparsity,
                               float(loss_scale), _ptr(scale_dev), _ptr(dsh), _ptr(ddensity), _ptr(loss), _stream()),
          "voxel_reg")


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


# ---- --random_bg (DESIGN.md §6f) ----------------------------------------------------------------------
def random_bg(seed, step, n_rays, device, step_dev=None):
    """[n_rays, 3] fp32 background colours in [0, 1) of training step ``step`` (or of step_dev[0], an int32 device
    scalar, when given): Philox4x32-10 keyed by ``seed``, counter (ray, step); the graph-captured step draws the same."""
    out = torch.empty(int(n_rays), 3, device=device, dtype=torch.float32)
    if step_dev is not None:
        _need_cuda(step_dev)
        if step_dev.dtype != torch.int32:
            raise TypeError("random_bg: step_dev must be int32")
    elif out.device.type != 'cuda':
        raise ValueError("random_bg draws on a CUDA device")
    check(load().ngp_random_bg(int(seed) & 0xFFFFFFFFFFFFFFFF, _ptr(step_dev) if step_dev is not None else None,
                               int(step), _ptr(out), int(n_rays), _stream()), "random_bg")
    return out


# ---- test-time evaluation --------------------------------------------------------------------------
def ssim(pred, target, height, width):
    """SSIM (torchmetrics' StructuralSimilarityIndexMeasure, data_range=1; DESIGN.md §6e) of fp32 images [H*W, 3]
    (one image) or [B, H*W, 3] -> fp32 [B] on the device.  Nothing is read back to the host."""
    _need_cuda(pred, target)
    if pred.dtype != torch.float32 or target.dtype != torch.float32:
        raise TypeError("ssim takes fp32 images")
    if pred.shape != target.shape:
        raise ValueError(f"ssim: pred {tuple(pred.shape)} and target {tuple(target.shape)} differ in shape")
    h, w = int(height), int(width)
    if pred.dim() not in (2, 3) or tuple(pred.shape[-2:]) != (h * w, 3):
        raise ValueError(f"ssim expects [H*W, 3] or [B, H*W, 3] with H*W = {h}*{w}, got {tuple(pred.shape)}")
    n = 1 if pred.dim() == 2 else pred.shape[0]
    p, t = pred.contiguous(), target.contiguous()
    partial = torch.empty(n * max(h - 10, 0), device=p.device, dtype=torch.float32)
    out = torch.empty(n, device=p.device, dtype=torch.float32)
    check(load().ngp_ssim(_ptr(p), _ptr(t), n, h, w, _ptr(partial), _ptr(out), _stream()), "ssim")
    return out


# ---- mesh export (DESIGN.md §6g) --------------------------------------------------------------------------------
def mesh_lattice_points(n, bound, start, count, bitfield, cascades, grid_size, scale):
    """World positions [count, 3] fp32 of lattice nodes [start, start + count) and their occupancy [count] uint8 (1:
    the node lies in an occupied cell by the marcher's position rule)."""
    _need_cuda(bitfield)
    xyz = torch.empty(int(count), 3, device=bitfield.device, dtype=torch.float32)
    occ = torch.empty(int(count), device=bitfield.device, dtype=torch.uint8)
    check(load().ngp_mesh_lattice_points(int(n), float(bound), int(start), int(count), _ptr(bitfield), int(cascades),
                                         int(grid_size), float(scale), _ptr(xyz), _ptr(occ), _stream()),
          "mesh_lattice_points")
    return xyz, occ


def mesh_lattice_store(sigma, occ, start, lattice):
    """lattice.view(-1)[start + j] = sigma[j] where occ[j] and sigma[j] is finite, else 0."""
    _need_cuda(sigma, occ, lattice)
    s = _f32c(sigma.reshape(-1))
    if occ.dtype != torch.uint8 or lattice.dtype != torch.float32 or not lattice.is_contiguous():
        raise TypeError("mesh_lattice_store: occ must be uint8 and lattice contiguous fp32")
    if s.numel() != occ.numel() or int(start) + s.numel() > lattice.numel():
        raise ValueError("mesh_lattice_store: sizes do not match the lattice")
    check(load().ngp_mesh_lattice_store(_ptr(s), _ptr(occ), int(start), s.numel(), _ptr(lattice), _stream()),
          "mesh_lattice_store")


class McStages:
    """The four marching-cubes launches of one fp32 lattice, so that each can be timed on its own; marching_cubes runs
    them in order."""

    def __init__(self, lattice, threshold, bound):
        _need_cuda(lattice)
        if lattice.dtype != torch.float32:
            raise TypeError("marching_cubes takes an fp32 lattice")
        n = lattice.shape[0]
        if lattice.dim() != 3 or tuple(lattice.shape) != (n, n, n) or not 2 <= n <= 1024:
            raise ValueError(f"marching_cubes expects an [N, N, N] lattice with 2 <= N <= 1024, got "
                             f"{tuple(lattice.shape)}")
        if not math.isfinite(threshold):
            raise ValueError(f"marching_cubes: the threshold must be finite, got {threshold}")
        if not (math.isfinite(bound) and bound > 0):
            raise ValueError(f"marching_cubes: the bound must be finite and > 0, got {bound}")
        self.lattice = lattice.contiguous()
        self.n, self.threshold, self.bound = n, float(threshold), float(bound)
        dev = lattice.device
        self.workspace = torch.empty(int(load().ngp_mc_workspace_bytes(n)), device=dev, dtype=torch.uint8)
        self.totals = torch.zeros(2, device=dev, dtype=torch.int64)
        self.vbase = None

    def count(self):
        check(load().ngp_mc_count(_ptr(self.lattice), self.n, self.threshold, _ptr(self.workspace), _stream()),
              "mc_count")

    def scan(self):
        check(load().ngp_mc_scan(self.n, _ptr(self.workspace), _ptr(self.totals), _stream()), "mc_scan")

    def sizes(self):
        """(V, F), read back to the host: the one synchronisation of the extraction."""
        v, f = (int(x) for x in self.totals.cpu())
        if v >= 2 ** 31 or f >= 2 ** 31:
            raise _lib.NgpError(f"marching_cubes: {v} vertices and {f} faces; both must stay below 2^31")
        return v, f

    def emit_vertices(self, n_vertices, vertices, normals):
        if self.vbase is None:
            self.vbase = torch.empty(self.n ** 3, device=self.lattice.device, dtype=torch.int32)
        check(load().ngp_mc_emit_vertices(_ptr(self.lattice), self.n, self.threshold, self.bound,
                                          _ptr(self.workspace), int(n_vertices), _ptr(self.vbase), _ptr(vertices),
                                          _ptr(normals), _stream()), "mc_emit_vertices")

    def emit_faces(self, n_faces, faces):
        check(load().ngp_mc_emit_faces(_ptr(self.lattice), self.n, self.threshold, _ptr(self.workspace),
                                       _ptr(self.vbase), int(n_faces), _ptr(faces), _stream()), "mc_emit_faces")


def marching_cubes(lattice, threshold, bound):
    """Marching cubes over an fp32 CUDA lattice [N, N, N] (indexed [ix, iy, iz], z fastest) spanning [-bound, bound]^3:
    (vertices [V, 3] fp32, normals [V, 3] fp32 unit, outward = toward lower values, faces [F, 3] int32 counter-clockwise
    seen from outside).  A node is inside when its value > threshold.  No mask, no model: DESIGN.md §6g."""
    st = McStages(lattice, threshold, bound)
    st.count()
    st.scan()
    nv, nf = st.sizes()
    dev = lattice.device
    vertices = torch.empty(nv, 3, device=dev, dtype=torch.float32)
    normals = torch.empty(nv, 3, device=dev, dtype=torch.float32)
    faces = torch.empty(nf, 3, device=dev, dtype=torch.int32)
    st.emit_vertices(nv, vertices, normals)
    st.emit_faces(nf, faces)
    st.vbase = None
    return vertices, normals, faces


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


# ---- camera extrinsics refinement (DESIGN.md §6i) ---------------------------------------------------------------
def _pose_buffers(*ts):
    for t in ts:
        if t.dtype != torch.float32 or not t.is_contiguous() or t.dim() != 2 or t.shape[1] != 8:
            raise TypeError("pose corrections, gradients and moments are contiguous fp32 [n_img, 8]")


def _img_index(img_idxs, n):
    i = img_idxs.to(torch.int64).reshape(-1)
    if i.numel() == 1 and n != 1:   # one image for the whole batch (--ray_sampling_strategy same_image)
        i = i.expand(n)
    if i.numel() != n:
        raise ValueError(f"{i.numel()} image indices for {n} rays")
    return i.contiguous()


def pose_apply(directions, img_idxs, poses, corr, rays_o=None, rays_d=None):
    """Rays (rays_o [n,3], rays_d [n,3] fp32) of camera directions [n,3] of images img_idxs [n] (or one index) under
    the corrected poses: R' = Exp(omega) R, o' = o + tau; poses [n_img, 3, 4], corr [n_img, 8]."""
    _need_cuda(directions, img_idxs, poses, corr, rays_o, rays_d)
    _pose_buffers(corr)
    d = _f32c(directions)
    n = d.shape[0]
    P = _f32c(poses)
    if P.dim() != 3 or tuple(P.shape[1:]) != (3, 4) or P.shape[0] != corr.shape[0]:
        raise ValueError(f"poses {tuple(P.shape)} must be [n_img, 3, 4] with n_img = {corr.shape[0]}")
    idx = _img_index(img_idxs, n)
    o = torch.empty(n, 3, device=d.device, dtype=torch.float32) if rays_o is None else rays_o
    dd = torch.empty(n, 3, device=d.device, dtype=torch.float32) if rays_d is None else rays_d
    check(load().ngp_pose_apply(_ptr(d), _ptr(idx), _ptr(P), _ptr(corr), P.shape[0], _ptr(o), _ptr(dd), n,
                                _stream()), "pose_apply")
    return o, dd


def pose_grad(dx, ts, rays_a, img_idxs, rays_d, grad, n_rays_dev=None, found_inf=None):
    """grad [n_img, 8] += per image (d' x G_d, 0, G_o, 0) of the rays in rays_a [n, 3] (ray, start, count), from
    the sample gradients dx [S, 3] and sample times ts [S]; img_idxs [n] (or one index) and rays_d [n, 3] by ray id."""
    _need_cuda(dx, ts, rays_a, img_idxs, rays_d, grad, n_rays_dev, found_inf)
    _pose_buffers(grad)
    if dx.dtype != torch.float32 or ts.dtype != torch.float32 or rays_a.dtype != torch.int32:
        raise TypeError("pose_grad: dx and ts are fp32, rays_a int32")
    n = rays_a.shape[0]
    idx = _img_index(img_idxs, n)
    dxc, tsc, d = dx.contiguous(), ts.contiguous(), _f32c(rays_d)
    if d.shape[0] != n or tsc.shape[0] != dxc.shape[0]:
        raise ValueError("pose_grad: rays_d needs one row per ray and ts one value per row of dx")
    check(load().ngp_pose_grad(_ptr(dxc), _ptr(tsc), _ptr(rays_a.contiguous()), _ptr(idx), _ptr(d), n,
                               _ptr(n_rays_dev), dxc.shape[0], grad.shape[0], _ptr(grad), _ptr(found_inf), _stream()),
          "pose_grad")


def pose_adam(corr, grad, exp_avg, exp_avg_sq, hyper, lr_ratio, found_inf=None, beta1=0.9, beta2=0.999, eps=1e-15):
    """One Adam step of the corrections with the model's device scalars ``hyper`` (ngp_adam_hyper_update) and a
    learning rate lr_ratio times the model's; the gradient goes through J_l(omega)^T first and is zeroed."""
    _need_cuda(corr, grad, exp_avg, exp_avg_sq, hyper, found_inf)
    _pose_buffers(corr, grad, exp_avg, exp_avg_sq)
    check(load().ngp_pose_adam(_ptr(corr), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(found_inf), _ptr(hyper),
                               float(lr_ratio), float(beta1), float(beta2), float(eps), corr.shape[0], _stream()),
          "pose_adam")


# ---- error-map ray sampling (DESIGN.md §6j) ---------------------------------------------------------------------
def _map_buffers(n_tiles, **ts):
    want = {"E": torch.int64, "acc": torch.int64, "cnt": torch.int32, "cdf": torch.int64}
    for k, t in ts.items():
        if t.dtype != want[k] or not t.is_contiguous() or t.numel() != n_tiles:
            raise TypeError(f"error map: {k} must be a contiguous {want[k]} tensor of {n_tiles} tiles")


def error_map_sample(cdf, geom, n_rays, seed, step=0, step_dev=None, out=None):
    """(img [n] int64, pix [n] int64, w [n] fp32) drawn from the map's CDF; geom = (n_img, W, H, R).  ``out`` = optional
    (img, pix, w) buffers to write (graph capture); ``step_dev`` an int32 device scalar read instead of ``step``."""
    _need_cuda(cdf, step_dev)
    n_img, W, H, R = (int(v) for v in geom)
    _map_buffers(n_img * R * R, cdf=cdf)
    if step_dev is not None and step_dev.dtype != torch.int32:
        raise TypeError("error_map_sample: step_dev must be int32")
    n = int(n_rays)
    if out is None:
        out = (torch.empty(n, device=cdf.device, dtype=torch.int64), torch.empty(n, device=cdf.device, dtype=torch.int64),
               torch.empty(n, device=cdf.device, dtype=torch.float32))
    img, pix, w = out
    check(load().ngp_error_map_sample(_ptr(cdf), n_img, W, H, R, int(seed) & 0xFFFFFFFFFFFFFFFF, _ptr(step_dev),
                                      int(step), _ptr(img), _ptr(pix), _ptr(w), n, _stream()), "error_map_sample")
    return img, pix, w


def error_map_accumulate(pred, target, img_idxs, pix_idxs, geom, acc, cnt, bg_rgb=None, alpha=None, b_load=1.0):
    """acc[t] += floor(min(sum_c (pred - target')^2, 3) 2^30), cnt[t] += 1 per ray; target' = target + (bg_rgb -
    b_load)(1 - alpha) when bg_rgb and alpha are given (the random-background head's target)."""
    _need_cuda(pred, target, img_idxs, pix_idxs, acc, cnt, bg_rgb, alpha)
    n_img, W, H, R = (int(v) for v in geom)
    _map_buffers(n_img * R * R, acc=acc, cnt=cnt)
    p, t = _f32c(pred), _f32c(target)
    n = p.shape[0]
    bg = None if bg_rgb is None else _f32c(bg_rgb)
    a = None if alpha is None else _f32c(alpha)
    ii, pi = img_idxs.to(torch.int64).contiguous(), pix_idxs.to(torch.int64).contiguous()
    if t.shape[0] != n or ii.numel() != n or pi.numel() != n or (bg is not None and bg.shape[0] != n) \
            or (a is not None and a.numel() != n):
        raise ValueError("error_map_accumulate: every per-ray input needs one row per ray")
    check(load().ngp_error_map_accumulate(_ptr(p), _ptr(t), _ptr(bg), _ptr(a), float(b_load), _ptr(ii), _ptr(pi),
                                          n_img, W, H, R, _ptr(acc), _ptr(cnt), n, _stream()), "error_map_accumulate")


def error_map_rebuild(E, acc, cnt, cdf, geom, ema_shift, floor_num, floor_den, workspace):
    """EMA of the interval's errors into E (acc, cnt cleared), masses and their inclusive scan into cdf."""
    _need_cuda(E, acc, cnt, cdf, workspace)
    n_img, W, H, R = (int(v) for v in geom)
    _map_buffers(n_img * R * R, E=E, acc=acc, cnt=cnt, cdf=cdf)
    check(load().ngp_error_map_rebuild(_ptr(E), _ptr(acc), _ptr(cnt), _ptr(cdf), n_img, W, H, R, int(ema_shift),
                                       int(floor_num), int(floor_den), _ptr(workspace),
                                       workspace.numel() * workspace.element_size(), _stream()), "error_map_rebuild")


def ray_grad_weight(rays_a, w, dsigmas, drgbs, found_inf=None, n_rows=None):
    """In place: every per-sample gradient of ray r (rows of rays_a [n, 3] = (ray, start, count)) times w[r]; dsigmas
    [S] fp32, drgbs [S, 3] fp32 or fp16.  found_inf (int32 [1], optional) is raised on a non-finite result."""
    _need_cuda(rays_a, w, dsigmas, drgbs, found_inf)
    if rays_a.dtype != torch.int32 or w.dtype != torch.float32 or dsigmas.dtype != torch.float32:
        raise TypeError("ray_grad_weight: rays_a int32, w and dsigmas fp32")
    for t in (rays_a, w, dsigmas, drgbs):
        if not t.is_contiguous():
            raise ValueError("ray_grad_weight: contiguous tensors only (the gradients are updated in place)")
    rows = dsigmas.shape[0] if n_rows is None else int(n_rows)
    check(load().ngp_ray_grad_weight(_ptr(rays_a), _ptr(w), _ptr(dsigmas), _ptr(drgbs), _tag(drgbs), _ptr(found_inf),
                                     rays_a.shape[0], rows, _stream()), "ray_grad_weight")


# ---- per-image exposure compensation (DESIGN.md §6k) ------------------------------------------------------------
def _exposure_buffers(*ts):
    for t in ts:
        if t.dtype != torch.float32 or not t.is_contiguous() or t.dim() != 2 or t.shape[1] != 4:
            raise TypeError("exposures, their gradient and moments are contiguous fp32 [n_img, 4]")


def _exposure_rows(rows, rays_a, what):
    if rays_a.dtype != torch.int32 or not rays_a.is_contiguous():
        raise TypeError(f"{what}: rays_a must be contiguous int32 [n, 3]")
    if rows.dim() != 2 or rows.shape[1] != 3 or not rows.is_contiguous():
        raise ValueError(f"{what}: rgb rows must be contiguous [S, 3]")


def exposure_apply(rgbs, rays_a, img_idxs, expo, out=None, n_rows_dev=None):
    """c' = 2^e[img(ray)] * c over every ray's rows of rgbs [S, 3] (fp16 or fp32) into a new buffer of the same dtype
    (or ``out``); rays_a [n, 3] int32 = (ray, start, count), img_idxs [n] (or one index) by ray id, expo [n_img, 4]."""
    _need_cuda(rgbs, rays_a, img_idxs, expo, out, n_rows_dev)
    _exposure_buffers(expo)
    _exposure_rows(rgbs, rays_a, "exposure_apply")
    n = rays_a.shape[0]
    idx = _img_index(img_idxs, n)
    out = torch.empty_like(rgbs) if out is None else out
    if out.dtype != rgbs.dtype or out.shape != rgbs.shape or out.data_ptr() == rgbs.data_ptr():
        raise ValueError("exposure_apply: out must be a separate buffer of rgbs' shape and dtype")
    check(load().ngp_exposure_apply(_ptr(rgbs), _tag(rgbs), _ptr(rays_a), _ptr(idx), _ptr(expo), expo.shape[0],
                                    _ptr(out), n, rgbs.shape[0], _ptr(n_rows_dev), _stream()), "exposure_apply")
    return out


def exposure_bwd(out, drgbs, rays_a, img_idxs, expo, grad, found_inf=None, n_rows_dev=None):
    """In place: drgbs [S, 3] = dL/dc' becomes dL/dc = g * dL/dc'; grad [n_img, 4] += ln2 * sum dL/dc' * c' per image,
    with out the rows exposure_apply wrote.  found_inf (int32 [1], optional) is raised on a non-finite result."""
    _need_cuda(out, drgbs, rays_a, img_idxs, expo, grad, found_inf, n_rows_dev)
    _exposure_buffers(expo, grad)
    _exposure_rows(drgbs, rays_a, "exposure_bwd")
    if out.dtype != drgbs.dtype or out.shape != drgbs.shape or not out.is_contiguous():
        raise ValueError("exposure_bwd: out and drgbs are contiguous rows of one shape and dtype")
    if grad.shape != expo.shape:
        raise ValueError("exposure_bwd: grad must have the exposures' shape")
    n = rays_a.shape[0]
    idx = _img_index(img_idxs, n)
    check(load().ngp_exposure_bwd(_ptr(out), _ptr(drgbs), _tag(drgbs), _ptr(rays_a), _ptr(idx), _ptr(expo),
                                  expo.shape[0], _ptr(grad), _ptr(found_inf), n, drgbs.shape[0], _ptr(n_rows_dev),
                                  _stream()), "exposure_bwd")


def exposure_adam(expo, grad, exp_avg, exp_avg_sq, hyper, lr_ratio, found_inf=None, beta1=0.9, beta2=0.999,
                  eps=1e-15):
    """One Adam step of the exposures with the model's device scalars ``hyper`` (ngp_adam_hyper_update) at lr_ratio
    times the model's learning rate, then the per-channel mean over the images subtracted; the gradient is zeroed."""
    _need_cuda(expo, grad, exp_avg, exp_avg_sq, hyper, found_inf)
    _exposure_buffers(expo, grad, exp_avg, exp_avg_sq)
    check(load().ngp_exposure_adam(_ptr(expo), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(found_inf),
                                   _ptr(hyper), float(lr_ratio), float(beta1), float(beta2), float(eps), expo.shape[0],
                                   _stream()), "exposure_adam")


# ---- camera intrinsics (DESIGN.md §6l) ---------------------------------------------------------------------------
def _camera_args(camera):
    """(model id, fp64 [8] host array) of a taichi_nerfs_b200.intrinsics.Camera."""
    return int(camera.model_id), (C.c_double * 8)(*[float(v) for v in camera.params])


def _intrinsics_buffer(t, rows, what):
    if t.dtype != torch.float32 or not t.is_contiguous() or t.dim() != 2 or t.shape[1] != 4 or \
            (rows is not None and t.shape[0] != rows):
        raise TypeError(f"{what} must be contiguous fp32 [{'n' if rows is None else rows}, 4]")


def camera_unproject(camera, W, H, pix_idxs=None, corr=None, out=None, grad_rows=None, n_bad=None, found_inf=None,
                     device=None):
    """Camera-frame directions [n, 3] fp32 (x_u, y_u, 1) of pixels pix_idxs [n] int64 of a W x H image, or of all W*H
    pixels of ``device`` when pix_idxs is None, under the corrections corr [1, 4] (or none).  grad_rows [n, 4]
    (optional) is zeroed; n_bad (int32 [1]) counts and found_inf (int32 [1]) flags the pixels that are not
    invertible."""
    dev = torch.device(device) if pix_idxs is None else pix_idxs.device
    if dev.type != "cuda":
        raise _lib.NgpError("libngp_b200 ops need CUDA tensors (there is no CPU fallback)")
    _need_cuda(pix_idxs, corr, out, grad_rows, n_bad, found_inf)
    if pix_idxs is not None and (pix_idxs.dtype != torch.int64 or not pix_idxs.is_contiguous()):
        raise TypeError("camera_unproject: pix_idxs must be contiguous int64")
    n = int(W) * int(H) if pix_idxs is None else pix_idxs.numel()
    if corr is not None:
        _intrinsics_buffer(corr, 1, "intrinsics corrections")
    if grad_rows is not None:
        _intrinsics_buffer(grad_rows, None, "camera_unproject: grad_rows")
        if grad_rows.shape[0] < n:
            raise ValueError(f"camera_unproject: grad_rows has {grad_rows.shape[0]} rows for {n} pixels")
    out = torch.empty(n, 3, device=dev, dtype=torch.float32) if out is None else out
    if out.dtype != torch.float32 or not out.is_contiguous() or out.numel() != 3 * n:
        raise ValueError(f"camera_unproject: out must be contiguous fp32 [{n}, 3]")
    model, params = _camera_args(camera)
    check(load().ngp_camera_unproject(_ptr(pix_idxs), n, int(W), int(H), model, params, _ptr(corr), _ptr(out),
                                      _ptr(grad_rows), _ptr(n_bad), _ptr(found_inf), _stream()), "camera_unproject")
    return out


def intrinsics_grad(dx, ts, rays_a, pix_idxs, img_idxs, poses, cam_dirs, camera, W, H, corr, grad_rays,
                    pose_corr=None, n_rays_dev=None, found_inf=None):
    """grad_rays[ray] [max_rays, 4] = (dL/da, dL/db_x, dL/db_y, 0) of every ray of rays_a [n, 3] (ray, start, count),
    from the sample gradients dx [S, 3] and times ts [S]; pix_idxs [n] (or more), img_idxs [n] (or one index) and
    cam_dirs [n, 3] (the unprojected directions the rays were formed with) by ray id; poses [n_img, 3, 4] with the
    extrinsics corrections pose_corr [n_img, 8] (or none).  Rows of rays without a rays_a row are left as they are."""
    _need_cuda(dx, ts, rays_a, pix_idxs, img_idxs, poses, cam_dirs, corr, grad_rays, pose_corr, n_rays_dev, found_inf)
    if dx.dtype != torch.float32 or ts.dtype != torch.float32 or rays_a.dtype != torch.int32:
        raise TypeError("intrinsics_grad: dx and ts are fp32, rays_a int32")
    if pix_idxs.dtype != torch.int64 or not pix_idxs.is_contiguous():
        raise TypeError("intrinsics_grad: pix_idxs must be contiguous int64")
    _intrinsics_buffer(corr, 1, "intrinsics corrections")
    _intrinsics_buffer(grad_rays, None, "intrinsics_grad: grad_rays")
    if pose_corr is not None:
        _pose_buffers(pose_corr)
    n = rays_a.shape[0]
    P = _f32c(poses)
    if P.dim() != 3 or tuple(P.shape[1:]) != (3, 4):
        raise ValueError(f"intrinsics_grad: poses {tuple(P.shape)} must be [n_img, 3, 4]")
    if pose_corr is not None and pose_corr.shape[0] != P.shape[0]:
        raise ValueError("intrinsics_grad: one pose correction per pose")
    rays = grad_rays.shape[0]
    idx = _img_index(img_idxs, rays)
    dxc, tsc, d = dx.contiguous(), ts.contiguous(), _f32c(cam_dirs)
    if d.shape[0] < rays or pix_idxs.numel() < rays or tsc.shape[0] != dxc.shape[0] or n > rays:
        raise ValueError("intrinsics_grad: cam_dirs and pix_idxs need a row per gradient row, ts one value per row of "
                         "dx, and grad_rays a row per ray")
    model, params = _camera_args(camera)
    check(load().ngp_intrinsics_grad(_ptr(dxc), _ptr(tsc), _ptr(rays_a.contiguous()), n, _ptr(n_rays_dev),
                                     dxc.shape[0], _ptr(pix_idxs), _ptr(idx), _ptr(P), _ptr(pose_corr), P.shape[0],
                                     _ptr(d), int(W), int(H), model, params, _ptr(corr), _ptr(grad_rays), rays,
                                     _ptr(found_inf), _stream()), "intrinsics_grad")


def intrinsics_adam(corr, grad_rays, n_rays, exp_avg, exp_avg_sq, hyper, lr_ratio, found_inf=None, beta1=0.9,
                    beta2=0.999, eps=1e-15, grad_out=None):
    """The sum of grad_rays[:n_rays] (fixed fp64 order, into grad_out [1, 4] when given), then one Adam step of corr
    [1, 4] with the model's device scalars ``hyper`` at lr_ratio times the model's learning rate (none when found_inf
    is raised)."""
    _need_cuda(corr, grad_rays, exp_avg, exp_avg_sq, hyper, found_inf, grad_out)
    for t, what in ((corr, "corrections"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        _intrinsics_buffer(t, 1, f"intrinsics {what}")
    if grad_out is not None:
        _intrinsics_buffer(grad_out, 1, "intrinsics_adam: grad_out")
    _intrinsics_buffer(grad_rays, None, "intrinsics_adam: grad_rays")
    if not 0 <= int(n_rays) <= grad_rays.shape[0]:
        raise ValueError(f"intrinsics_adam: n_rays {n_rays} outside [0, {grad_rays.shape[0]}]")
    check(load().ngp_intrinsics_adam(_ptr(corr), _ptr(grad_rays), int(n_rays), _ptr(exp_avg), _ptr(exp_avg_sq),
                                     _ptr(found_inf), _ptr(hyper), float(lr_ratio), float(beta1), float(beta2),
                                     float(eps), _ptr(grad_out), _stream()), "intrinsics_adam")


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


def _voxel_block(block, field, *others):
    """(G, C, host block6) of a voxel field [G, G, G, C] and its node block B.  The kernels derive every offset from G
    and C, so anything but a 4-D cube (and companions of the same shape) is refused."""
    if field.dim() != 4 or not field.shape[0] == field.shape[1] == field.shape[2]:
        raise ValueError(f"a voxel field is [G, G, G, C], got {tuple(field.shape)}")
    for t in others:
        if t.shape != field.shape:
            raise ValueError(f"voxel buffers differ in shape: {tuple(t.shape)} vs {tuple(field.shape)}")
    G, C_ = int(field.shape[0]), int(field.shape[-1])
    return G, C_, (C.c_int32 * 6)(*[int(v) for v in block])


def check_finite_voxel_block(grad, block, found_inf):
    """found_inf[0] = 1 when an element of the voxel-field gradient grad [G,G,G,C] inside the node block ``block`` =
    (lo_x, lo_y, lo_z, hi_x, hi_y, hi_z) is not finite (``layout.voxel_reg_block``)."""
    _voxel_inputs(grad)
    _need_cuda(found_inf)
    G, C_, b6 = _voxel_block(block, grad)
    check(load().ngp_check_finite_voxel_block(_ptr(grad), G, C_, b6, _ptr(found_inf), _stream()),
          "check_finite_voxel_block")


def adam_step_voxel_block(param, grad, exp_avg, exp_avg_sq, block, hyper, found_inf=None, beta1=0.9, beta2=0.999,
                          eps=1e-15):
    """ngp_adam_step_dyn (device scalars ``hyper``, zero_grad) over the elements of a voxel field [G,G,G,C] inside the
    node block ``block``; everything outside it is left alone."""
    _voxel_inputs(param, grad, exp_avg, exp_avg_sq, hyper)
    _need_cuda(found_inf)
    G, C_, b6 = _voxel_block(block, param, grad, exp_avg, exp_avg_sq)
    check(load().ngp_adam_step_voxel_block_dyn(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), G, C_, b6,
                                               _ptr(found_inf), _ptr(hyper), float(beta1), float(beta2), float(eps),
                                               _stream()), "adam_step_voxel_block")


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
