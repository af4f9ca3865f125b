"""Host-side multiresolution hash-grid layout.

Restates what the reference derives in ``HashEncoder.__init__``
(modules/hash_encoder.py:157-208, modules/hash_encoder_half.py:230-284 and the
helpers modules/utils.py:19-42): the per-level resolution, table size, offset and
the first level that needs the xor-prime hash.  In addition it precomputes, in
fp32 semantics, the per-level ``scale`` / ``resolution`` that the Taichi kernel
recomputes per thread (modules/hash_encoder.py:73-80,103-104) so that the CPU
oracle and the CUDA kernels consume literally the same numbers (SURVEY.md §7
"hard part 2": an ``expf`` that is 1 ulp high changes the dense stride).
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, field
from typing import List

import numpy as np

NGP_MAX_LEVELS = 16


class CHashLayout(ctypes.Structure):
    """ctypes mirror of ``ngp_hash_layout`` (include/ngp_b200.h)."""

    _fields_ = [
        ("n_levels", ctypes.c_int32),
        ("feat_dim", ctypes.c_int32),
        ("begin_fast_hash_level", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("offsets", ctypes.c_int32 * NGP_MAX_LEVELS),
        ("map_sizes", ctypes.c_int32 * NGP_MAX_LEVELS),
        ("scales", ctypes.c_float * NGP_MAX_LEVELS),
        ("resolutions", ctypes.c_uint32 * NGP_MAX_LEVELS),
    ]


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def _f32(x: float) -> float:
    return float(np.float32(x))


@dataclass
class HashLayout:
    levels: int
    feat_dim: int
    base_res: float
    max_res: float
    max_params: int
    log_b: float = 0.0
    offsets: List[int] = field(default_factory=list)
    map_sizes: List[int] = field(default_factory=list)
    layout_res: List[int] = field(default_factory=list)   # f64 resolution used for sizing
    scales: List[float] = field(default_factory=list)     # f32 kernel scale
    resolutions: List[int] = field(default_factory=list)  # f32 kernel resolution
    begin_fast_hash_level: int = 0
    total_entries: int = 0

    @property
    def total_param_size(self) -> int:
        return self.total_entries * self.feat_dim

    @property
    def out_dim(self) -> int:
        return self.levels * self.feat_dim

    def as_ctypes(self) -> CHashLayout:
        c = CHashLayout()
        c.n_levels = self.levels
        c.feat_dim = self.feat_dim
        c.begin_fast_hash_level = self.begin_fast_hash_level
        for i in range(self.levels):
            c.offsets[i] = self.offsets[i]
            c.map_sizes[i] = self.map_sizes[i]
            c.scales[i] = self.scales[i]
            c.resolutions[i] = self.resolutions[i]
        return c


def growth_log_b(base_res: float, max_res: float, levels: int) -> float:
    """log(max_res/base_res)/(levels-1) in f64 (modules/utils.py:31-39); 0 for a single level."""
    return math.log(float(max_res) / float(base_res)) / float(levels - 1) if levels > 1 else 0.0


def level_scale_f32(lvl: int, log_b: float, base_res: float):
    """(scale, resolution) of one level as the Taichi kernels compute them in f32 (modules/hash_encoder.py:73-80,
    modules/triplane.py:27-33): exp of the f32 product, correctly rounded to f32; f32 multiply by base_res; f32
    subtract 1; resolution = u32(ceil(scale)) + 1."""
    arg = _f32(_f32(float(lvl)) * _f32(log_b))
    e = _f32(math.exp(arg))
    scale = _f32(_f32(_f32(float(base_res)) * e) - 1.0)
    return scale, int(math.ceil(scale)) + 1


def make_hash_layout(max_params: int = 2 ** 19, levels: int = 16, base_res: float = 16.0,
                     max_res: float = 2048.0, feature_per_level: int = 2) -> HashLayout:
    levels = int(levels)
    if not 1 <= levels <= NGP_MAX_LEVELS:
        raise ValueError(f"levels must be in [1, {NGP_MAX_LEVELS}], got {levels}")
    max_params = int(max_params)
    lay = HashLayout(levels=levels, feat_dim=int(feature_per_level), base_res=float(base_res),
                     max_res=float(max_res), max_params=max_params)
    lay.log_b = growth_log_b(base_res, max_res, levels)

    offset = 0
    first_hashed = levels
    for lvl in range(levels):
        # sizing uses f64 (modules/utils.py:19-29)
        res = math.ceil(float(base_res) * math.exp(float(lvl) * lay.log_b) - 1.0) + 1
        full = res ** 3
        size = min(max_params, _round_up(full, 8))
        lay.layout_res.append(int(res))
        lay.offsets.append(offset)
        lay.map_sizes.append(int(size))
        if full > size and first_hashed == levels:
            first_hashed = lvl
        offset += size

        scale, res32 = level_scale_f32(lvl, lay.log_b, base_res)
        lay.scales.append(scale)
        lay.resolutions.append(res32)

    lay.begin_fast_hash_level = first_hashed
    lay.total_entries = offset
    return lay


# ---- tri-plane encoder (modules/triplane.py of the reference) ------------------------------------------
NGP_TRIPLANE_MAX_RES = 16384


class CTriplaneLayout(ctypes.Structure):
    """ctypes mirror of ``ngp_triplane_layout`` (include/ngp_b200.h)."""

    _fields_ = [
        ("n_levels", ctypes.c_int32),
        ("feat_dim", ctypes.c_int32),
        ("max_res", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("scales", ctypes.c_float * NGP_MAX_LEVELS),
        ("resolutions", ctypes.c_uint32 * NGP_MAX_LEVELS),
    ]


@dataclass
class TriplaneLayout:
    levels: int
    feat_dim: int
    base_res: float
    max_res: int
    log_b: float = 0.0
    scales: List[float] = field(default_factory=list)     # f32 kernel scale
    resolutions: List[int] = field(default_factory=list)  # f32 kernel resolution

    @property
    def total_param_size(self) -> int:
        # three max_res^2 planes of F features (triplane.py:126-128)
        return self.max_res ** 2 * 3 * self.feat_dim

    @property
    def out_dim(self) -> int:
        return self.levels * self.feat_dim

    def as_ctypes(self) -> CTriplaneLayout:
        c = CTriplaneLayout()
        c.n_levels = self.levels
        c.feat_dim = self.feat_dim
        c.max_res = self.max_res
        for i in range(self.levels):
            c.scales[i] = self.scales[i]
            c.resolutions[i] = self.resolutions[i]
        return c


def make_triplane_layout(levels: int = 16, base_res: float = 16.0, max_res: int = 2048,
                         feature_per_level: int = 2) -> TriplaneLayout:
    """Per-level constants of TriPlaneEncoder (modules/triplane.py:103-136): the same f64 growth factor and f32
    scale / resolution as the hash levels.  Supported: levels 1..16, F in {2, 4}, integer max_res in
    [2, 16384]."""
    levels, F = int(levels), int(feature_per_level)
    if not 1 <= levels <= NGP_MAX_LEVELS:
        raise ValueError(f"levels must be in [1, {NGP_MAX_LEVELS}], got {levels}")
    if F not in (2, 4):
        raise ValueError(f"feature_per_level must be 2 or 4 for the tri-plane encoder, got {F}")
    if int(max_res) != max_res or not 2 <= int(max_res) <= NGP_TRIPLANE_MAX_RES:
        raise ValueError(f"max_res must be an integer in [2, {NGP_TRIPLANE_MAX_RES}], got {max_res}")
    lay = TriplaneLayout(levels=levels, feat_dim=F, base_res=float(base_res), max_res=int(max_res))
    lay.log_b = growth_log_b(base_res, max_res, levels)
    for lvl in range(levels):
        scale, res = level_scale_f32(lvl, lay.log_b, base_res)
        lay.scales.append(scale)
        lay.resolutions.append(res)
    return lay


# ---- voxel grid (VoxelGrid of the reference, modules/networks.py:382-575) -------------------------------
NGP_VOXEL_MAX_GRID = 2048
VOXEL_SH_DEGREES = (0, 1, 2)


class CVoxelLayout(ctypes.Structure):
    """ctypes mirror of ``ngp_voxel_layout`` (include/ngp_b200.h)."""

    _fields_ = [
        ("grid", ctypes.c_int32),
        ("sh_degree", ctypes.c_int32),
        ("radius", ctypes.c_float),
        ("c_min", ctypes.c_float),
    ]


@dataclass
class VoxelLayout:
    grid: int
    sh_degree: int
    radius: float   # fp32 node spacing
    c_min: float    # fp32 world coordinate of node 0 on every axis

    @property
    def sh_dim(self) -> int:
        return (1 + self.sh_degree) ** 2

    @property
    def channels(self) -> int:
        """sh channels per node (3 colours x sh_dim); the density is a field of its own."""
        return 3 * self.sh_dim

    def as_ctypes(self) -> CVoxelLayout:
        return CVoxelLayout(self.grid, self.sh_degree, self.radius, self.c_min)


def voxel_node_offset(grid: int) -> int:
    """Lattice index of the node at the origin: node i sits at (i - ceil(G/2) + 1) * radius (networks.py:458-463)."""
    return int(math.ceil(grid / 2)) - 1


def make_voxel_layout(grid_size: int = 256, grid_radius: float = 0.0125, sh_degree: int = 2) -> VoxelLayout:
    """Kernel constants of a VoxelGrid: c_min = (1 - ceil(G/2)) * radius (the minimum node coordinate,
    networks.py:521-522), computed in f64 and rounded once to f32.  Supported: G in [1, 2048], sh_degree 0..2."""
    G, deg = int(grid_size), int(sh_degree)
    if G != grid_size or not 1 <= G <= NGP_VOXEL_MAX_GRID:
        raise ValueError(f"grid_size must be an integer in [1, {NGP_VOXEL_MAX_GRID}], got {grid_size}")
    if deg != sh_degree or deg not in VOXEL_SH_DEGREES:
        raise ValueError(f"sh_degree must be 0, 1 or 2, got {sh_degree}")
    if not (math.isfinite(grid_radius) and grid_radius > 0):
        raise ValueError(f"grid_radius must be positive and finite, got {grid_radius}")
    return VoxelLayout(grid=G, sh_degree=deg, radius=_f32(grid_radius),
                       c_min=_f32(-voxel_node_offset(G) * float(grid_radius)))
