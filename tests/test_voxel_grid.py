"""CPU checks of the voxel-grid model (`--model_name svox`): command line, model config, parameters and buffers, the
lattice against the reference's formulas, the SH basis of the fp64 restatement, the layout and the C-ABI's argument
validation."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import voxel_ref as R
from taichi_nerfs_b200.layout import make_voxel_layout


def _opts(*args):
    from opt import get_opts
    return get_opts(list(args))


def test_opt_accepts_svox_and_refuses_combinations():
    h = _opts('--model_name', 'svox', '--sh_degree', '1', '--grid_size', '64')
    assert (h.model_name, h.sh_degree, h.grid_size) == ('svox', 1, 64)
    for extra in (['--encoder_type', 'triplane'], ['--graph_step'], ['--deployment']):
        with pytest.raises(SystemExit):
            _opts('--model_name', 'svox', *extra)
    assert _opts().model_name == 'ngp'
    for flag in ('--sh_degree', '--grid_size', '--grid_radius', '--origin_sh', '--origin_sigma'):
        from opt import _FLAGS
        assert 'unused' not in dict(_FLAGS)[flag]['help']


def test_build_model_config_returns_voxel_grid_arguments():
    from modules.networks import MODEL_DICT
    from modules.voxel_grid import VoxelGrid
    from train import build_model_config
    h = _opts('--model_name', 'svox', '--sh_degree', '0', '--grid_size', '33', '--grid_radius', '0.03',
              '--origin_sh', '0.25', '--origin_sigma', '0.5', '--half_opt')
    cfg = build_model_config(h)
    assert cfg == {'scale': 0.5, 'half_opt': True, 'sh_degree': 0, 'grid_size': 33, 'grid_radius': 0.03,
                   'origin_sh': 0.25, 'origin_sigma': 0.5}
    assert MODEL_DICT['svox'] is VoxelGrid
    m = MODEL_DICT[h.model_name](**cfg)
    assert (m.field_size, m.sh_degree, m.grid_size) == (33, 0, 128)
    # an ngp configuration is unchanged
    assert build_model_config(_opts())['pos_encoder_type'] == 'hash'


def test_state_dict_keys_shapes_and_fill():
    from modules.voxel_grid import VoxelGrid
    m = VoxelGrid(sh_degree=1, grid_size=5, origin_sh=0.5, origin_sigma=0.25)
    sd = m.state_dict()
    assert set(sd) == {'sh_fields', 'density_fields', 'center', 'xyz_min', 'xyz_max', 'half_size',
                       'density_bitfield', 'density_grid', 'grid_coords'}
    assert sd['sh_fields'].shape == (5, 5, 5, 12) and sd['sh_fields'].dtype == torch.float32
    assert sd['density_fields'].shape == (5, 5, 5, 1) and sd['density_fields'].dtype == torch.float32
    assert torch.all(sd['sh_fields'] == 0.5) and torch.all(sd['density_fields'] == 0.25)
    # the occupancy grid is NGP's, whatever the field resolution
    assert m.grid_size == 128 and m.cascades == 1
    assert sd['density_grid'].shape == (1, 128 ** 3) and sd['density_bitfield'].shape == (128 ** 3 // 8,)
    assert sd['grid_coords'].shape == (128 ** 3, 3)
    assert [n for n, _ in m.named_parameters()] == ['sh_fields', 'density_fields']
    assert not hasattr(m, 'pos_encoder') and m._fusable(torch.zeros(1, 3)) is False
    with torch.device('meta'):
        d = VoxelGrid()          # the default 256^3 degree-2 field: 470 M parameters
    assert d.sh_fields.shape == (256, 256, 256, 27) and d.density_fields.shape == (256, 256, 256, 1)
    assert sum(p.numel() for p in d.parameters()) == 256 ** 3 * 28


def test_ngp_buffers_unchanged():
    from modules.networks import NGP
    m = NGP(max_res=1024)
    keys = list(m.state_dict())
    assert keys[:7] == ['center', 'xyz_min', 'xyz_max', 'half_size', 'density_bitfield', 'density_grid',
                        'grid_coords']
    assert m.grid_size == 128 and m.cascades == 1 and m.scale == 0.5


@pytest.mark.parametrize("sh_degree", [-1, 3, 4])
def test_unsupported_degree_raises(sh_degree):
    from modules.voxel_grid import VoxelGrid
    with pytest.raises(ValueError):
        VoxelGrid(sh_degree=sh_degree, grid_size=2)


@pytest.mark.parametrize("G", [2, 5, 96, 97, 256])
def test_node_coordinates_match_reference_formula(G):
    """networks.py:450-466: meshgrid of arange(G) per axis, minus np.ceil(G/2) - 1, times grid_radius."""
    from modules.voxel_grid import VoxelGrid
    radius = 0.0125
    i = np.arange(G)
    cx, cy, cz = np.meshgrid(i, i, i, indexing='ij')
    ref = np.stack([cx - np.ceil(G / 2) + 1, cy - np.ceil(G / 2) + 1, cz - np.ceil(G / 2) + 1], -1) * radius
    ref = ref.reshape(-1, 3)
    lat = R.lattice(G, radius).numpy()
    ours = np.stack(np.meshgrid(lat, lat, lat, indexing='ij'), -1).reshape(-1, 3)
    np.testing.assert_allclose(ours, ref, rtol=0, atol=1e-15)
    with torch.device('meta') if G == 256 else torch.device('cpu'):
        m = VoxelGrid(grid_size=G, grid_radius=radius, sh_degree=0)
    np.testing.assert_array_equal(m.lattice().numpy(), lat)
    lay = make_voxel_layout(G, radius, 0)
    # c_min = the smallest node coordinate (networks.py:522, grid_normalized_coords.min(0)), rounded to fp32
    assert lay.c_min == float(np.float32(ref.min()))
    assert lay.radius == float(np.float32(radius))


@pytest.mark.parametrize("deg", [0, 1, 2])
def test_sh_basis_orthonormal_on_sphere(deg):
    """Gauss-Legendre in cos(theta) x uniform in phi integrates polynomials of degree <= 4 on the sphere exactly."""
    t, wt = np.polynomial.legendre.leggauss(8)
    P = 16
    phi = 2 * np.pi * np.arange(P) / P
    ct, ph = np.meshgrid(t, phi, indexing='ij')
    st = np.sqrt(1 - ct ** 2)
    d = torch.from_numpy(np.stack([st * np.cos(ph), st * np.sin(ph), ct], -1).reshape(-1, 3))
    w = torch.from_numpy((wt[:, None] * np.full(P, 2 * np.pi / P)[None, :]).reshape(-1))
    Y = R.sh_basis(deg, d)
    gram = (Y * w[:, None]).T @ Y
    assert Y.shape[1] == (deg + 1) ** 2
    np.testing.assert_allclose(gram.numpy(), np.eye((deg + 1) ** 2), atol=1e-12)


def test_reference_interpolation_hand_worked():
    """G = 2, radius 1: nodes at 0 and 1 on every axis.  Field value at node (i,j,k) = 4i + 2j + k: a linear
    function, which trilinear interpolation reproduces inside the cell; outside, missing corners read zero."""
    f = torch.tensor([[[[4. * i + 2 * j + k] for k in range(2)] for j in range(2)] for i in range(2)],
                     dtype=torch.float64)
    xyz = torch.tensor([[0.25, 0.5, 0.75], [0., 0., 0.], [1., 1., 1.], [1.5, 0., 0.], [-0.5, 0, 0], [9, 9, 9]],
                       dtype=torch.float64)
    out = R.interpolate(xyz, f, 1.0, 0.0)[:, 0]
    want = torch.tensor([4 * 0.25 + 2 * 0.5 + 0.75, 0., 7., 0.5 * 4, 0.5 * 0., 0.], dtype=torch.float64)
    torch.testing.assert_close(out, want, rtol=0, atol=1e-15)


def test_cabi_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib
    L = _lib.load()
    lay = make_voxel_layout(4, 0.25, 2).as_ctypes()
    f = C.c_void_p(16)
    assert L.ngp_voxel_fwd(f, f, f, f, C.byref(lay), f, f, 0, None) == 0       # n = 0: nothing to do
    assert L.ngp_voxel_fwd(f, f, f, f, C.byref(lay), f, f, -1, None) != 0
    assert L.ngp_voxel_fwd(None, f, f, f, C.byref(lay), f, f, 1, None) != 0
    assert L.ngp_voxel_fwd(f, f, f, f, None, f, f, 1, None) != 0
    assert L.ngp_voxel_bwd(f, f, f, f, f, f, C.byref(lay), f, f, 1, None, 2, None) != 0   # unknown mapping
    assert L.ngp_voxel_bwd(f, f, f, f, f, f, C.byref(lay), None, f, 1, None, 0, None) != 0
    for bad in (dict(sh_degree=3), dict(grid=0), dict(grid=4096), dict(radius=0.0), dict(radius=math.inf)):
        b = make_voxel_layout(4, 0.25, 2).as_ctypes()
        for k, v in bad.items():
            setattr(b, k, v)
        assert L.ngp_voxel_fwd(f, f, f, f, C.byref(b), f, f, 1, None) != 0, bad
    assert b"radius" in L.ngp_last_error()
