"""CPU checks of the tri-plane encoder (modules/triplane.py of the reference): the oracle against an independent
numpy restatement and a hand-worked value, its backward against finite differences, the layout, the model / CLI
wiring and the C-ABI's argument validation."""
import ctypes as C
import math

import numpy as np
import pytest

from taichi_nerfs_b200.layout import make_hash_layout, make_triplane_layout
from triplane_ref import triplane_numpy


@pytest.fixture(scope="module")
def O():
    from oracle import triplane
    triplane.build()
    return triplane


def _positions(rng, n, lay):
    """Random points, points on cell boundaries of every level, the corners 0 and 1."""
    pts = [rng.random((n, 3), dtype=np.float32)]
    for level in range(lay.levels):
        r = lay.resolutions[level]
        k = rng.integers(0, r, (16, 3))
        pts.append(((k.astype(np.float32) + np.float32(0.5)) / np.float32(r - 1)).clip(0, 1).astype(np.float32))
    pts.append(np.array([[0, 0, 0], [1, 1, 1], [0, 1, 0.5], [1, 0, 1]], np.float32))
    return np.concatenate(pts)


@pytest.mark.parametrize("levels,F,max_res", [(8, 4, 1024), (16, 2, 2048)])
def test_oracle_forward_equals_numpy_restatement(O, levels, F, max_res):
    rng = np.random.default_rng(levels * F)
    lay = make_triplane_layout(levels, 16, max_res, F)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    xyz = _positions(rng, 3000, lay)
    got = O.triplane_encode_fwd(xyz, table, lay)
    want = triplane_numpy(xyz, table, lay)
    assert got.shape == (xyz.shape[0], levels * F)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


def test_known_answer_level0():
    """x = (0.5, 0.25, 0.75), L=8 F=4 max_res=1024, level 0: res = 16, pos = x*15 + 0.5 = (8, 4.25, 11.75).
    max_res-grid coordinates u32(g/16 * 1023): g=4 -> 255, 5 -> 319, 8 -> 511, 9 -> 575, 11 -> 703, 12 -> 767.
    plane 0 (x, y), weights (1-0)(1-.25) = .75 at (511, 255) and (1-0)(.25) = .25 at (511, 319):
        lf0 = .75*[1,2,3,4] + .25*[5,6,7,8] = [2,3,4,5]
    plane 1 (y, z): the four corners (255|319, 703|767) all hold 2, weights sum to 1: lf1 = 2
    plane 2 (z, x): (1-.75)*1 at (703, 511) = 4 and .75*1 at (767, 511) = 8: lf2 = 1 + 6 = 7
    out[:, j*8 + 0] = lf0*lf1*lf2 = [28, 42, 56, 70].  A swapped plane pair, the hash's [level][F] column order or a
    rounded (not truncated) grid mapping all read zeros instead."""
    from oracle import triplane as O
    lay = make_triplane_layout(8, 16, 1024, 4)
    assert lay.resolutions[0] == 16
    mr, F = 1024, 4
    table = np.zeros(lay.total_param_size, np.float32)

    def put(fd, u, v, vals):
        e = fd * mr * mr * F + (u + v * mr) * F
        table[e:e + F] = vals

    put(0, 511, 255, [1, 2, 3, 4])
    put(0, 511, 319, [5, 6, 7, 8])
    for u in (255, 319):
        for v in (703, 767):
            put(1, u, v, 2.0)
    put(2, 703, 511, 4.0)
    put(2, 767, 511, 8.0)
    out = O.triplane_encode_fwd(np.array([[0.5, 0.25, 0.75]], np.float32), table, lay)
    np.testing.assert_array_equal(out[0, [0, 8, 16, 24]], [28, 42, 56, 70])
    np.testing.assert_array_equal(triplane_numpy(np.array([[0.5, 0.25, 0.75]], np.float32), table, lay)[0, [0, 8, 16, 24]],
                                  [28, 42, 56, 70])


def test_oracle_forward_clamps_outside_unit_cube(O):
    """Positions outside [0, 1] (no bound check in the reference, triplane.py:88-89) stay inside the table: the
    max_res-grid coordinate is clamped.  Inside [0, 1] the clamp changes nothing (test above)."""
    lay = make_triplane_layout(8, 16, 64, 4)
    rng = np.random.default_rng(1)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    near = np.array([[1.001, 0.5, 0.5], [0.5, -0.001, 1.0005], [1.0, 1.0, 1.0001]], np.float32)
    far = np.array([[1.5, 2.0, -0.5], [-1e30, 1e30, np.inf], [np.nan, 0.5, 0.5]], np.float32)
    out = O.triplane_encode_fwd(near, table, lay)
    want = triplane_numpy(near, table, lay, clamp=True)
    np.testing.assert_array_equal(out.view(np.uint32), want.view(np.uint32))
    assert np.isfinite(out).all()
    assert np.isfinite(O.triplane_encode_fwd(far[:1], table, lay)).all()
    O.triplane_encode_fwd(far, table, lay)   # defined (saturating casts + clamp): no read outside the table


def test_oracle_backward_matches_finite_differences(O):
    """The loss sum(dout * fwd) is linear in each table entry, so fp64 central differences of the fp64 restatement
    are exact up to rounding."""
    lay = make_triplane_layout(4, 4, 32, 4)
    rng = np.random.default_rng(5)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    xyz = rng.random((12, 3), dtype=np.float32)
    dout = rng.standard_normal((12, lay.out_dim)).astype(np.float32)
    dout[3] = 0.0
    g = O.triplane_encode_bwd(xyz, table, dout, lay)
    t64 = table.astype(np.float64)
    touched = np.flatnonzero(g)
    assert touched.size > 100
    pick = np.concatenate([rng.choice(touched, 60, replace=False),
                           rng.choice(np.setdiff1d(np.arange(g.size), touched), 20, replace=False)])
    h = 1e-3
    for e in pick:
        tp, tm = t64.copy(), t64.copy()
        tp[e] += h
        tm[e] -= h
        fd = ((dout * triplane_numpy(xyz, tp, lay, np.float64)).sum()
              - (dout * triplane_numpy(xyz, tm, lay, np.float64)).sum()) / (2 * h)
        assert abs(g[e] - fd) <= 1e-5 * np.abs(g).max() + 1e-6 * abs(fd), (e, g[e], fd)


def test_triplane_layout():
    lay = make_triplane_layout(8, 16, 1024, 4)
    assert lay.log_b == math.log(1024 / 16) / 7
    assert lay.out_dim == 32
    assert lay.total_param_size == 12_582_912
    assert make_triplane_layout(8, 16, 4096, 4).total_param_size == 201_326_592
    # the hash levels' fp32 scale / resolution derivation, shared
    h = make_hash_layout(2 ** 19, 8, 16, 1024, 4)
    assert lay.scales == h.scales and lay.resolutions == h.resolutions
    assert lay.resolutions[0] == 16 and lay.resolutions[-1] == 1024
    c = lay.as_ctypes()
    assert (c.n_levels, c.feat_dim, c.max_res) == (8, 4, 1024)
    for bad in (dict(levels=17), dict(levels=0), dict(feature_per_level=3), dict(max_res=1)):
        kw = dict(levels=8, base_res=16, max_res=1024, feature_per_level=4)
        kw.update(bad)
        with pytest.raises(ValueError):
            make_triplane_layout(**kw)


def test_cli_and_model_build_on_cpu():
    import torch
    from modules.networks import NGP
    from opt import get_opts
    hp = get_opts(['--encoder_type', 'triplane'])
    assert hp.encoder_type == 'triplane'
    import train
    cfg = train.build_model_config(hp)
    assert cfg['pos_encoder_type'] == 'triplane' and cfg['max_res'] == 1024
    for extra in (['--half_opt'], ['--graph_step'], ['--deployment']):
        with pytest.raises(SystemExit):
            get_opts(['--encoder_type', 'triplane'] + extra)
    torch.manual_seed(0)
    m = NGP(**cfg)
    enc = m.pos_encoder
    assert type(enc).__name__ == 'TriPlaneEncoder'
    assert (enc.levels, enc.feature_per_level, enc.base_res, enc.max_res) == (8, 4, 16, 1024)
    assert enc.out_dim == 32 and enc.total_param_size == 12_582_912
    assert enc.log_b == math.log(1024 / 16) / 7
    sd = m.state_dict()
    assert 'pos_encoder.plane_embedding' in sd and not any('hash' in k for k in sd)
    p = sd['pos_encoder.plane_embedding']
    assert p.dtype == torch.float32 and p.shape == (12_582_912,)
    assert 0.0 <= float(p.min()) and float(p.max()) < 1.0   # U[0, 1) (triplane.py:136)
    assert m.xyz_encoder.input_dim == 32


def test_cabi_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    lib = _lib.load()
    lay = make_triplane_layout(8, 16, 1024, 4).as_ctypes()
    x = (C.c_float * 3)()
    assert lib.ngp_triplane_encode_fwd(None, None, C.byref(lay), None, 8, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert lib.ngp_triplane_encode_fwd(x, None, None, x, 8, None, None) < 0
    bad = make_triplane_layout(8, 16, 1024, 4).as_ctypes()
    bad.feat_dim = 3
    assert lib.ngp_triplane_encode_fwd(x, x, C.byref(bad), x, 8, None, None) < 0
    assert b"feature" in lib.ngp_last_error()
    bad = make_triplane_layout(8, 16, 1024, 4).as_ctypes()
    bad.n_levels = 17
    assert lib.ngp_triplane_encode_bwd(x, x, x, C.byref(bad), x, 8, None) < 0
    assert lib.ngp_triplane_encode_fwd_dyn(x, x, C.byref(bad), x, 8, None, None, None) < 0
    assert lib.ngp_triplane_encode_bwd(None, None, None, C.byref(lay), None, 8, None) < 0
    assert lib.ngp_triplane_encode_fwd(x, x, C.byref(lay), x, -1, None, None) < 0
    # n = 0 is a no-op success
    assert lib.ngp_triplane_encode_fwd(None, None, C.byref(lay), None, 0, None, None) == 0
    assert lib.ngp_triplane_encode_fwd_dyn(None, None, C.byref(lay), None, 0, None, None, None) == 0
    assert lib.ngp_triplane_encode_bwd(None, None, None, C.byref(lay), None, 0, None) == 0


def test_ops_refuse_cpu_tensors():
    import torch
    from taichi_nerfs_b200 import _lib, ops
    lay = make_triplane_layout(8, 16, 64, 4)
    with pytest.raises(_lib.NgpError):
        ops.triplane_encode_fwd(torch.zeros(4, 3), torch.zeros(lay.total_param_size), lay.as_ctypes())
    with pytest.raises(_lib.NgpError):
        ops.triplane_encode_bwd(torch.zeros(4, 3), torch.zeros(lay.total_param_size), torch.zeros(4, 32),
                                lay.as_ctypes(), torch.zeros(lay.total_param_size))
