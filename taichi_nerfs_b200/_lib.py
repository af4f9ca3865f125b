"""ctypes loader for libngp_b200.so — the only way the Python host code reaches the GPU kernels.

The product path has NO CPU fallback: if the shared library is missing (or a call is made
without a CUDA device) an exception is raised.  The CPU oracle under oracle/ is test
infrastructure and is never imported from here.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

from .layout import CHashLayout, CTriplaneLayout, CVoxelLayout

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libngp_b200.so")

F32, F16 = 0, 1

_lock = threading.Lock()
_lib = None


class MlpWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1", "w2", "w3", "w4", "w5")]


class NgpError(RuntimeError):
    pass


def _declare(lib):
    i64, i32, f32, vp, ci = C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_int
    lay = C.POINTER(CHashLayout)
    tri = C.POINTER(CTriplaneLayout)
    vox = C.POINTER(CVoxelLayout)
    mw = C.POINTER(MlpWeights)
    sigs = {
        "ngp_version": (ci, []),
        "ngp_last_error": (C.c_char_p, []),
        "ngp_launch_count": (i64, []),
        "ngp_ray_aabb_intersect": (ci, [vp, vp, f32, vp, i64, vp]),
        "ngp_raymarching_train_count": (ci, [vp, vp, vp, vp, vp, ci, ci, f32, f32, ci, vp, vp, i64, vp]),
        "ngp_raymarching_train_write": (ci, [vp, vp, vp, vp, vp, ci, ci, f32, f32, vp, vp, vp, vp, vp, vp, i64, i64, vp]),
        "ngp_raymarching_frame": (ci, [vp, vp, vp, vp, vp, ci, ci, f32, f32, ci, vp, vp, vp, vp, vp, vp, i64, i64, vp]),
        "ngp_raymarching_test": (ci, [vp, vp, vp, vp, vp, ci, ci, f32, f32, ci, vp, vp, vp, vp, vp, i64, vp]),
        "ngp_hash_encode_fwd": (ci, [vp, vp, lay, vp, ci, i64, vp]),
        "ngp_hash_encode_bwd": (ci, [vp, vp, ci, lay, vp, i64, vp]),
        "ngp_hash_encode_bwd_input": (ci, [vp, vp, vp, ci, lay, vp, i64, vp]),
        "ngp_hash_encode_bwd_input_dyn": (ci, [vp, vp, vp, ci, lay, vp, i64, vp, vp, vp]),
        "ngp_hash_encode_fwd_dyn": (ci, [vp, vp, lay, vp, ci, i64, vp, vp, vp]),
        "ngp_hash_encode_bwd_dyn": (ci, [vp, vp, ci, lay, vp, i64, vp, vp, vp]),
        "ngp_hash_encode_bwd_levels": (ci, [vp, vp, ci, lay, vp, i64, vp, vp, ci, ci, vp, vp]),
        "ngp_hash_bwd_level_groups": (ci, [lay, ci, ci, i64, vp]),
        "ngp_triplane_encode_fwd": (ci, [vp, vp, tri, vp, i64, vp, vp]),
        "ngp_triplane_encode_fwd_dyn": (ci, [vp, vp, tri, vp, i64, vp, vp, vp]),
        "ngp_triplane_encode_bwd": (ci, [vp, vp, vp, tri, vp, i64, vp]),
        "ngp_triplane_encode_bwd_dyn": (ci, [vp, vp, vp, tri, vp, i64, vp, vp, vp, vp]),
        "ngp_voxel_fwd": (ci, [vp, vp, vp, vp, vox, vp, vp, i64, vp]),
        "ngp_voxel_fwd_dyn": (ci, [vp, vp, vp, vp, vox, vp, vp, i64, vp, vp]),
        "ngp_voxel_bwd": (ci, [vp, vp, vp, vp, vp, vp, vox, vp, vp, i64, vp, ci, vp]),
        "ngp_voxel_bwd_dyn": (ci, [vp, vp, vp, vp, vp, vp, vox, vp, vp, i64, vp, vp, vp]),
        "ngp_voxel_reg": (ci, [vp, vp, vox, vp, f32, f32, f32, f32, vp, vp, vp, vp, vp]),
        "ngp_mlp_fwd_dyn": (ci, [vp, ci, vp, mw, vp, vp, vp, i64, vp, vp]),
        "ngp_mlp_bwd_dyn": (ci, [vp, ci, vp, mw, vp, vp, vp, vp, vp, i64, vp, vp, vp]),
        "ngp_adam_step_dyn": (ci, [vp, vp, vp, vp, vp, vp, vp, f32, f32, f32, ci, i64, vp]),
        "ngp_adam_hyper_update": (ci, [vp, f32, f32, i32, f32, f32, f32, vp, vp, vp]),
        "ngp_loss_scale_update": (ci, [vp, vp, f32, f32, i32, f32, vp, ci, vp]),
        "ngp_step_reset": (ci, [vp, vp, vp, vp, vp]),
        "ngp_mse_loss_grad_dyn": (ci, [vp, vp, vp, f32, vp, vp, vp, vp, i64, vp]),
        "ngp_mse_loss_grad": (ci, [vp, vp, vp, f32, f32, vp, vp, vp, i64, vp]),
        "ngp_dir_encode": (ci, [vp, vp, i64, vp]),
        "ngp_mlp_save_bytes": (i64, [i64]),
        "ngp_mlp_fwd": (ci, [vp, ci, vp, mw, vp, vp, vp, i64, vp]),
        "ngp_mlp_bwd": (ci, [vp, ci, vp, mw, vp, vp, vp, vp, vp, i64, vp]),
        "ngp_composite_train_fwd": (ci, [vp, vp, ci, vp, vp, vp, f32, vp, vp, vp, vp, vp, i64, i64, vp]),
        "ngp_composite_train_bwd": (ci, [vp, vp, vp, vp, vp, vp, ci, vp, vp, vp, vp, vp, vp, f32, vp, vp, i64, i64, vp]),
        "ngp_composite_test": (ci, [vp, vp, ci, vp, vp, vp, vp, f32, vp, vp, vp, i64, vp]),
        "ngp_ray_head_fused": (ci, [vp, vp, ci, vp, vp, vp, f32, f32, vp, f32, vp, vp, vp, vp, vp, i64, vp]),
        "ngp_ray_head_fused_distortion": (ci, [vp, vp, ci, vp, vp, vp, vp, f32, f32, vp, f32, f32, vp, vp, vp, vp, vp,
                                               i64, vp]),
        "ngp_random_bg": (ci, [C.c_uint64, vp, i32, vp, i64, vp]),
        "ngp_ray_head_fused_random_bg": (ci, [vp, vp, ci, vp, vp, vp, vp, vp, vp, f32, f32, vp, f32, f32, vp, vp, vp,
                                              vp, vp, i64, vp]),
        "ngp_ray_head_fused_depth": (ci, [vp, vp, ci, vp, vp, vp, vp, f32, vp, vp, f32, f32, vp, f32, f32, vp, f32, vp,
                                          vp, vp, vp, vp, i64, vp]),
        "ngp_distortion_fwd": (ci, [vp, vp, vp, vp, vp, i64, i64, vp]),
        "ngp_distortion_bwd": (ci, [vp, vp, vp, vp, vp, vp, i64, i64, vp]),
        "ngp_ssim": (ci, [vp, vp, i64, ci, ci, vp, vp, vp]),
        "ngp_packbits": (ci, [vp, f32, vp, i64, vp]),
        "ngp_packbits_dev": (ci, [vp, vp, f32, vp, i64, vp]),
        "ngp_sample_ray_batch": (ci, [vp, ci, vp, vp, i64, i64, vp, vp, i64, C.c_uint64, vp, i32,
                                      vp, vp, vp, vp, vp, vp, i64, vp]),
        "ngp_morton3d": (ci, [vp, vp, i64, vp]),
        "ngp_morton3d_invert": (ci, [vp, vp, i64, vp]),
        "ngp_adam_step": (ci, [vp, vp, vp, vp, vp, vp, f32, f32, f32, f32, f32, i32, ci, i64, vp]),
        "ngp_check_finite": (ci, [vp, i64, vp, vp]),
        "ngp_check_finite_voxel_block": (ci, [vp, i32, i32, vp, vp, vp]),
        "ngp_adam_step_voxel_block_dyn": (ci, [vp, vp, vp, vp, i32, i32, vp, vp, vp, f32, f32, f32, vp]),
        "ngp_grad_pack_f16": (ci, [vp, vp, i64, vp]),
        "ngp_check_finite_f16": (ci, [vp, i64, vp, vp]),
        "ngp_adam_step_dyn_g16": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, f32, f32, f32, i64, vp]),
        "ngp_p2p_alloc": (ci, [i64, C.POINTER(vp), vp]),
        "ngp_p2p_open": (ci, [vp, C.POINTER(vp)]),
        "ngp_p2p_close": (ci, [vp]),
        "ngp_p2p_free": (ci, [vp]),
        "ngp_p2p_flag_bytes": (i64, []),
        "ngp_p2p_barrier": (ci, [vp, ci, ci, vp, vp, vp]),
        "ngp_adam_step_p2p": (ci, [vp, vp, vp, vp, vp, ci, ci, vp, vp, f32, f32, f32, i64, i64, i64, i64, vp]),
        "ngp_frame_begin": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, i64, vp]),
        "ngp_frame_round_begin": (ci, [vp, vp]),
        "ngp_raymarching_round": (ci, [vp, vp, vp, vp, ci, ci, f32, f32, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                       i64, i64, vp]),
        "ngp_composite_round": (ci, [vp, vp, ci, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, vp, i64, ci, vp]),
        "ngp_grid_workspace_bytes": (i64, [ci, ci]),
        "ngp_grid_sample_cells": (ci, [vp, ci, ci, f32, f32, ci, i64, C.c_uint64, C.c_uint32, vp, vp, vp, vp]),
        "ngp_grid_update": (ci, [vp, vp, vp, i64, ci, ci, vp, f32, f32, vp, vp, vp, vp]),
        "ngp_mesh_lattice_points": (ci, [i64, f32, i64, i64, vp, ci, ci, f32, vp, vp, vp]),
        "ngp_mesh_lattice_store": (ci, [vp, vp, i64, i64, vp, vp]),
        "ngp_mc_workspace_bytes": (i64, [i64]),
        "ngp_mc_count": (ci, [vp, i64, f32, vp, vp]),
        "ngp_mc_scan": (ci, [i64, vp, vp, vp]),
        "ngp_mc_emit_vertices": (ci, [vp, i64, f32, f32, vp, i64, vp, vp, vp, vp]),
        "ngp_mc_emit_faces": (ci, [vp, i64, f32, vp, vp, i64, vp, vp]),
        "ngp_pose_apply": (ci, [vp, vp, vp, vp, i64, vp, vp, i64, vp]),
        "ngp_pose_grad": (ci, [vp, vp, vp, vp, vp, i64, vp, i64, i64, vp, vp, vp]),
        "ngp_pose_adam": (ci, [vp, vp, vp, vp, vp, vp, f32, f32, f32, f32, i64, vp]),
        "ngp_camera_unproject": (ci, [vp, i64, i64, i64, ci, vp, vp, vp, vp, vp, vp, vp]),
        "ngp_intrinsics_grad": (ci, [vp, vp, vp, i64, vp, i64, vp, vp, vp, vp, i64, vp, i64, i64, ci, vp, vp, vp, i64,
                                     vp, vp]),
        "ngp_intrinsics_adam": (ci, [vp, vp, i64, vp, vp, vp, vp, f32, f32, f32, f32, vp, vp]),
        "ngp_error_map_workspace_bytes": (i64, [i64]),
        "ngp_error_map_sample": (ci, [vp, i64, i64, i64, i64, C.c_uint64, vp, i32, vp, vp, vp, i64, vp]),
        "ngp_error_map_accumulate": (ci, [vp, vp, vp, vp, f32, vp, vp, i64, i64, i64, i64, vp, vp, i64, vp]),
        "ngp_error_map_rebuild": (ci, [vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, ci, vp, i64, vp]),
        "ngp_ray_grad_weight": (ci, [vp, vp, vp, vp, ci, vp, i64, i64, vp]),
        "ngp_exposure_apply": (ci, [vp, ci, vp, vp, vp, i64, vp, i64, i64, vp, vp]),
        "ngp_exposure_bwd": (ci, [vp, vp, ci, vp, vp, vp, i64, vp, vp, i64, i64, vp, vp]),
        "ngp_exposure_adam": (ci, [vp, vp, vp, vp, vp, vp, f32, f32, f32, f32, i64, vp]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    return sigs


EXPORTS = None


def load():
    """Load (once) and return the C-ABI library.  Raises if it has not been built."""
    global _lib, EXPORTS
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise NgpError(
                        f"{LIB_PATH} not found: build it with `python -m taichi_nerfs_b200.build` "
                        "(there is no CPU fallback for the product path)")
                lib = C.CDLL(LIB_PATH)
                EXPORTS = _declare(lib)
                _lib = lib
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().ngp_last_error().decode("utf-8", "replace")
        raise NgpError(f"{what or 'libngp_b200'} failed (rc={rc}): {msg}")


def launch_count() -> int:
    return int(load().ngp_launch_count())
