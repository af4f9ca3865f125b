"""CPU checks of the voxel-grid regularisers (`--tv_sigma_loss_w`, `--tv_sh_loss_w`, `--sparsity_loss_w`): the flags,
the C-ABI's argument validation, the host computation of the node block B, and fault injection for the fp64
comparator that tests/test_gpu_voxel_reg.py judges the kernel by."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import voxel_reg_ref as RR
from taichi_nerfs_b200.layout import make_voxel_layout, voxel_reg_block

FLAGS = ('--tv_sigma_loss_w', '--tv_sh_loss_w', '--sparsity_loss_w')


def _opts(*args):
    from opt import get_opts
    return get_opts(list(args))


def test_flags_defaults_svox_only_and_refusals():
    from opt import _FLAGS
    h = _opts()
    assert (h.tv_sigma_loss_w, h.tv_sh_loss_w, h.sparsity_loss_w) == (0.0, 0.0, 0.0)
    for flag in FLAGS:
        assert 'svox only' in dict(_FLAGS)[flag]['help']
        assert getattr(_opts('--model_name', 'svox', flag, '0.25'), flag[2:]) == 0.25
        assert getattr(_opts(flag, '0'), flag[2:]) == 0.0          # a zero weight is fine with ngp
        for bad in (('--model_name', 'ngp', flag, '0.1'), ('--model_name', 'svox', flag, '-0.1'),
                    ('--model_name', 'svox', flag, 'nan'), ('--model_name', 'svox', flag, 'inf')):
            with pytest.raises(SystemExit):
                _opts(*bad)


def _lay_block(G, radius, scale):
    lay = make_voxel_layout(G, radius, 0)
    return lay, voxel_reg_block(lay, scale)


def _u32(lay, x):
    f = np.float32
    return float(f(f(f(x) - f(lay.c_min)) / f(lay.radius)))


@pytest.mark.parametrize("G,radius,scale", [(256, 0.0125, 0.5), (255, 0.0125, 0.5), (97, 0.03, 0.5), (96, 0.03, 0.5),
                                            (97, 0.03, 2.0), (8, 0.3, 0.5), (2, 0.3, 0.5), (1, 0.0125, 0.5),
                                            (256, 0.0125, 0.1), (33, 0.05, 0.7)])
def test_block_bounds(G, radius, scale):
    """B = floor(u(-scale)) - 1 .. floor(u(scale)) + 2 per axis, clamped to [0, G-1]; it contains the fp32 floor(u)
    and floor(u) + 1 of both box faces wherever those are nodes."""
    lay, b = _lay_block(G, radius, scale)
    lo, hi = b[0], b[3]
    assert b[:3] == (lo,) * 3 and b[3:] == (hi,) * 3 and 0 <= lo < hi <= G
    fl_lo, fl_hi = math.floor(_u32(lay, -scale)), math.floor(_u32(lay, scale))
    assert lo == max(fl_lo - 1, 0) and hi == min(fl_hi + 2, G - 1) + 1
    for x in (-scale, scale):
        f = math.floor(_u32(lay, x))
        for node in (f, f + 1):
            if 0 <= node < G:
                assert lo <= node < hi, (x, node, b)


def test_block_hand_worked():
    # shipped lattice: c_min = -127 * 0.0125 = -1.5875; u(-0.5) = 87, u(0.5) = 167 -> nodes 86 .. 169: 84 per axis
    lay, b = _lay_block(256, 0.0125, 0.5)
    assert b == (86, 86, 86, 170, 170, 170)
    # odd G: c_min = -48 * 0.03 = -1.44; u(-0.5) = 31.33, u(0.5) = 64.67 -> 30 .. 66
    assert _lay_block(97, 0.03, 0.5)[1] == (30,) * 3 + (67,) * 3
    # a box larger than the lattice: the whole grid; a single node
    assert _lay_block(97, 0.03, 2.0)[1] == (0,) * 3 + (97,) * 3
    assert _lay_block(1, 0.0125, 0.5)[1] == (0,) * 3 + (1,) * 3
    # G = 2, radius 0.3: nodes at 0 and 0.3, u(-0.5) = -1.67 -> clamped to 0; u(0.5) = 1.67 -> 3, clamped to 1
    assert _lay_block(2, 0.3, 0.5)[1] == (0,) * 3 + (2,) * 3


def test_voxel_grid_stores_block():
    from modules.voxel_grid import VoxelGrid
    m = VoxelGrid(sh_degree=0, grid_size=33, grid_radius=0.05, scale=0.7)
    assert m._reg_block == voxel_reg_block(make_voxel_layout(33, 0.05, 0), 0.7)
    assert set(m.state_dict()) == {'sh_fields', 'density_fields', 'center', 'xyz_min', 'xyz_max', 'half_size',
                                   'density_bitfield', 'density_grid', 'grid_coords'}


def test_trainer_refuses_voxel_reg_without_voxel_fields_and_bad_weights():
    from modules.networks import NGP
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.trainer import NGPTrainer
    with pytest.raises(ValueError, match="voxel fields"):
        NGPTrainer(NGP(max_res=1024), voxel_reg=(1.0, 0.0, 0.0))
    for bad in ((-1.0, 0.0, 0.0), (0.0, math.nan, 0.0), (0.0, 0.0, math.inf), (1.0, 1.0)):
        with pytest.raises(ValueError, match="voxel_reg"):
            NGPTrainer(VoxelGrid(sh_degree=0, grid_size=4), voxel_reg=bad)


def test_cabi_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib
    L = _lib.load()
    lay = make_voxel_layout(8, 0.25, 1).as_ctypes()
    f = C.c_void_p(16)

    def call(block=(1, 1, 1, 7, 7, 7), w=(1.0, 1.0, 1.0), scale=1.0, scale_dev=None, ptrs=(f, f, f, f), layout=lay):
        b6 = None if block is None else (C.c_int32 * 6)(*block)
        sh, den, dsh, dden = ptrs
        return L.ngp_voxel_reg(sh, den, None if layout is None else C.byref(layout), b6, *w, scale, scale_dev, dsh,
                               dden, None, None)

    assert call(w=(0.0, 0.0, 0.0)) == 0                          # all weights 0: nothing to do
    assert call(w=(0.0, 0.0, 0.0), ptrs=(None,) * 4) == 0
    assert call(layout=None) != 0
    assert call(block=None) != 0
    for bad in ((0, 0, 0, 0, 8, 8), (-1, 0, 0, 8, 8, 8), (0, 0, 0, 8, 8, 9), (3, 0, 0, 2, 8, 8), (0, 5, 0, 8, 5, 8)):
        assert call(block=bad) != 0, bad
    assert b"block" in L.ngp_last_error()
    for w in ((-1.0, 0.0, 0.0), (0.0, -0.5, 0.0), (0.0, 0.0, math.nan), (math.inf, 0.0, 0.0)):
        assert call(w=w) != 0, w
    assert b"weights" in L.ngp_last_error()
    assert call(scale=math.inf) != 0 and call(scale=math.nan) != 0
    for i in range(4):
        ptrs = [f] * 4
        ptrs[i] = None
        assert call(ptrs=tuple(ptrs)) != 0
    assert b"null" in L.ngp_last_error()
    bad = make_voxel_layout(8, 0.25, 1).as_ctypes()
    bad.sh_degree = 3
    assert call(layout=bad) != 0


# ---- fault injection for the comparator -----------------------------------------------------------------------------
def _case(seed=7, G=12, deg=1, block=(2, 1, 3, 11, 10, 12)):
    """Fields with flat patches (s = sqrt(eps)), a patch of tiny differences (D^2 ~ eps) and densities on a 1/8
    grid on both sides of 0; a non-cubic block that touches the grid's end on z."""
    rng = np.random.default_rng(seed)
    D3 = 3 * (deg + 1) ** 2
    sh = (rng.integers(-8, 9, (G, G, G, D3)) / 8).astype(np.float32)
    sh[4:7, 4:7, 4:7] = 0.25
    sh[7:11, 2:6, 5:9] = (0.5 + rng.integers(0, 3, (4, 4, 4, D3)) * 2.0 ** -13).astype(np.float32)
    den = (rng.integers(-8, 9, (G, G, G, 1)) / 8).astype(np.float32)
    den[5:10, 5:10, 5:10] = (rng.integers(0, 3, (5, 5, 5, 1)) * 2.0 ** -13).astype(np.float32)
    den[2:4, 2:4, 2:4] = 0.0
    pre_sh = rng.standard_normal(sh.shape).astype(np.float32) * 1e-3
    pre_den = rng.standard_normal(den.shape).astype(np.float32) * 1e-3
    return sh, den, block, pre_sh, pre_den


WEIGHTS = (0.7, 1.3, 0.4)
SCALE = 2.0 ** 10


def _run_np(fault=None, weights=WEIGHTS):
    sh, den, block, pre_sh, pre_den = _case()
    dsh, dden = pre_sh.copy(), pre_den.copy()
    RR.kernel_np(sh, den, block, weights, SCALE, dsh, dden, fault=fault)
    t = torch.from_numpy
    return RR.check(RR.block_of(t(dsh), block), RR.block_of(t(dden), block), RR.block_of(t(pre_sh), block),
                    RR.block_of(t(pre_den), block), RR.block_of(t(sh), block), RR.block_of(t(den), block), weights,
                    SCALE, what=f"numpy fault={fault}"), (dsh, dden, pre_sh, pre_den, block)


def test_comparator_accepts_numpy_fp32_copy():
    (L, worst), (dsh, dden, pre_sh, pre_den, block) = _run_np()
    assert 0 < worst <= 1 and L > 0
    # outside B nothing moved
    mask = np.ones(dsh.shape[:3], bool)
    mask[tuple(slice(a, b) for a, b in zip(block[:3], block[3:]))] = False
    assert np.array_equal(dsh[mask], pre_sh[mask]) and np.array_equal(dden[mask], pre_den[mask])
    for w in ((0.0, 1.0, 0.0), (1.0, 0.0, 0.0), (0.0, 0.0, 1.0)):
        _run_np(weights=w)


@pytest.mark.parametrize("fault", RR.FAULTS)
def test_comparator_rejects_planted_mistakes(fault):
    with pytest.raises(AssertionError, match="off the fp64 bound"):
        _run_np(fault=fault)
