"""The hash encoder's entry points that the parity and step tests leave loose, one kernel at a time on fixed inputs,
against a plain high-precision reference (tests/hash_ref.py).

A. Table backward (F = 2) at the garden layout, max_res 4096: train.py's resolution for every scene with
   scale != 0.5.  Levels 14 and 15 (resolutions 2831 and 4096) are the only ones where the fp16 kernel's
   pos -= f16(pos_grid) (hash_encoder_half.py:132) has an effect: an odd grid coordinate above 2048 rounds to an even
   neighbour, the fraction leaves [0, 1) and some trilinear weights are negative.  Checked by level group against
   the fp64 scatter, plain and with the AABB folded in and the row count read on the device (_dyn).
B. The generic-width kernels (every F != 2): the --deployment model's L=4 F=4 dense layout, a hashed F=4 layout and
   F = 1, 3, 8.  Forward bit-exact against the oracle (whose generic-F forward is itself checked here against the
   independent numpy restatement of tests/test_oracle.py); backward against the fp64 scatter; both plain and _dyn.
C. Input gradient dL/dx, fp32 and fp16, at max_res 1024 and 4096, against the exact derivative of the forward in
   fp64: in fp16 that is the derivative of the forward's fraction p - f16(g), not of p - g.  The CPU oracle is held
   to the same reference.
D. Argument validation of these entry points (CPU only).

Tolerances, each from the error model of the operation:
- table backward: every entry within (k + 4) u (|prefill| + sum |w dy|), u = 2^-24, k = contributions to the entry.
  Each contribution is one fp32 product (exact when contracted) and k + 1 operands are summed in some order, so
  (k + 1) u bounds any atomic order; entries outside the launched levels, and entries no sample reaches, must be
  bit-unchanged.  Rows whose dy is zero at every level carry NaN positions, so a kernel that scattered them instead
  of skipping them would leave NaN in the table.
- dL/dx on the GPU: every component within (8L + 8) u sum |term| (sum over the 8L level-corner terms of
  scale * (|t0 dy0| + |t1 dy1|) * |w_a w_b|).  Per term the kernel rounds the two products and their sum (2u
  relative to |t0 dy0| + |t1 dy1|), the product with scale, the two factors 1 - pos and the two products with them
  (5u): 7u; the sequential sum of 8L terms adds (8L - 1) u.  Total (8L + 6) u plus second-order terms.
- dL/dx of the oracle: 4u sum |term|.  It rounds each factor 1 - pos to fp32 (2u per term) and the fp64 result to
  fp32 (u); its fp64 arithmetic adds ~8L 2^-53.
Every reference is finite and every bound is written as `err <= bound`, so a NaN or inf result fails.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from taichi_nerfs_b200.layout import make_hash_layout

from hash_ref import (PAD, U, _aabb6, _check_scatter, _level_ranges, _level_slice, _normalise, _ray_points,
                      _world_points, grid_cell, n_dev_cases, np_hash_bwd_f64, np_hash_dx_f64, rows_of)

DEV = "cuda"
F32, F16 = 0, 1


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def ST():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def chk(rc):
    from taichi_nerfs_b200 import _lib
    _lib.check(rc)


def i32(v):
    return torch.tensor([v], device=DEV, dtype=torch.int32)


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


@functools.lru_cache(maxsize=None)
def _layout(args):
    return make_hash_layout(*args)


@functools.lru_cache(maxsize=2)
def _table(args, half):
    rng = np.random.default_rng(list(args) + [half])
    t = rng.standard_normal(_layout(args).total_param_size).astype(np.float32)
    return (t * 0.1).astype(np.float16) if half else t


def _unit_points(rng, n):
    """Uniform points of [0, 1]^3 with the corners, face centres and one point in seven on a face (exactly 0 or 1)."""
    return _normalise(_world_points(rng, n, 0.5), 0.5)


def _on_faces(rng, x):
    """The first rows moved to the cube's corners and one row in seven moved onto a face."""
    x = x.copy()
    corners = np.array([[(c >> d) & 1 for d in range(3)] for c in range(8)], np.float32)
    k = min(len(x), 8)
    x[:k] = corners[:k]
    idx = rng.choice(len(x), len(x) // 7, replace=False)
    x[idx, rng.integers(0, 3, idx.size)] = (rng.random(idx.size) < 0.5).astype(np.float32)
    return x


def _dout(rng, n, lay, half):
    """dL/demb with skipped rows (all-zero dy), single (row, level) pairs with an all-zero dy, and (row, level) pairs
    with some features zero and others not: those must still contribute."""
    L, F = lay.levels, lay.feat_dim
    d = rng.standard_normal((n, L, F)).astype(np.float32)
    d[rng.random(n) < 0.1] = 0.0
    d[rng.random((n, L)) < 0.05] = 0.0
    d[(rng.random((n, L)) < 0.1)[:, :, None] & (rng.random((n, L, F)) < 0.5)] = 0.0
    d = d.reshape(n, L * F)
    return d.astype(np.float16) if half else d


def _poison_skipped_rows(rng, x, dout, lay):
    """NaN positions on some rows whose dy is zero at every level: a kernel that did not skip them would scatter NaN."""
    dead = np.flatnonzero(~np.asarray(dout).reshape(len(x), -1).astype(bool).any(1))
    assert dead.size > 0
    x = x.copy()
    x[rng.choice(dead, min(dead.size, 16), replace=False)] = np.nan
    return x


def _assert_dout_mix(dout, lay, n_rows):
    """The inputs hold skipped rows, skipped (row, level) pairs and, for F > 1, partly zero ones."""
    nz = np.asarray(dout[:n_rows]).reshape(n_rows, lay.levels, lay.feat_dim) != 0
    assert (~nz.any((1, 2))).any() and (~nz.any(2) & nz.any(2).any(1, keepdims=True)).any()
    if lay.feat_dim > 1:
        assert (nz.any(2) & ~nz.all(2)).any()


# ---- A. table backward at the garden layout -------------------------------------------------------------------------
GARDEN = (2 ** 19, 16, 16, 4096, 2)
GARDEN_SCALE = 16.0
GARDEN_GROUPS = dict(_level_ranges(_layout(GARDEN)), levels_14_15=(14, 16))


def _assert_fp16_cast_exercised(xn, lay):
    """Levels 14 and 15: some rows have an odd grid coordinate above 2048, and some fp16 fractions lie outside
    [0, 1).  Without both, the fp16 and fp32 grid casts would agree on these inputs."""
    x = xn[np.isfinite(xn).all(1)]
    assert lay.resolutions[14] > 2048
    for lvl in (14, 15):
        g, frac = grid_cell(x, lay, lvl, True)
        assert ((g > 2048) & (g % 2 == 1)).any(), f"level {lvl}: no odd grid coordinate above 2048"
        assert ((frac < 0) | (frac >= 1)).any(), f"level {lvl}: every fp16 fraction is in [0, 1)"


def _garden_ray_points(rng, n):
    """Ray samples one finest cell (1/4096) apart, with corner and face points."""
    return _on_faces(rng, _ray_points(rng, n, per_ray=200, step=1.0 / 4096))


def test_garden_inputs_exercise_the_fp16_grid_cast():
    lay = _layout(GARDEN)
    _assert_fp16_cast_exercised(_garden_ray_points(np.random.default_rng(40), 20000), lay)
    rng = np.random.default_rng(41)
    _assert_fp16_cast_exercised(_normalise(_world_points(rng, 3000, GARDEN_SCALE), GARDEN_SCALE), lay)


@functools.lru_cache(maxsize=1)
def _garden_bwd_case(half):
    lay = _layout(GARDEN)
    rng = np.random.default_rng(42 + half)
    n = 20000
    xn = _garden_ray_points(rng, n)
    dout = _dout(rng, n, lay, half)
    xn = _poison_skipped_rows(rng, xn, dout, lay)
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    return xn, dout, prefill, np_hash_bwd_f64(xn, dout, lay, half, range(lay.levels))


@pytest.mark.gpu
@pytest.mark.parametrize("group", list(GARDEN_GROUPS))
@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_garden_levels_fp64_bound(lib, half, group):
    lay = _layout(GARDEN)
    cl = lay.as_ctypes()
    a, b = GARDEN_GROUPS[group]
    xn, dout, prefill, (ref, mag, cnt) = _garden_bwd_case(half)
    _assert_fp16_cast_exercised(xn, lay)
    _assert_dout_mix(dout, lay, len(xn))
    g, t_x, t_d = T(prefill), T(xn), T(dout)
    chk(lib.ngp_hash_encode_bwd_levels(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), len(xn), None, None,
                                       a, b, None, ST()))
    lo, hi = _level_slice(lay, a, b)
    assert cnt[lo:hi].max() > 1   # the run accumulation is exercised
    _check_scatter(N(g), prefill, ref, mag, cnt, lo, hi, f"levels [{a},{b})")


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_garden_dyn_aabb(lib, half):
    """Garden-box world positions normalised inside the kernel, the row count read on the device: rows at or beyond
    min(n_max, n_dev) contribute nothing."""
    _garden_bwd_case.cache_clear()     # the level-group tests' reference is not needed here
    s = GARDEN_SCALE
    lay = _layout(GARDEN)
    cl = lay.as_ctypes()
    rng = np.random.default_rng(44 + half)
    n_max = 3000
    xn = _garden_ray_points(rng, n_max + PAD)
    dout = _dout(rng, n_max + PAD, lay, half)
    xw = (xn * np.float32(2 * s) - np.float32(s)).astype(np.float32)
    xw[n_max // 2: n_max // 2 + n_max // 7] = _world_points(rng, n_max // 7, s)       # face points too
    xw = _poison_skipped_rows(rng, xw, dout, lay)
    xnn = _normalise(xw, s)
    _assert_fp16_cast_exercised(xnn[:n_max // 2], lay)
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    t_x, t_d = T(xw), T(dout)
    ref_m = ref = None
    for nd in n_dev_cases(n_max):
        g = T(prefill)
        chk(lib.ngp_hash_encode_bwd_levels(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n_max,
                                           P(i32(nd)), _aabb6(s), 0, lay.levels, None, ST()))
        m = rows_of(nd, n_max)
        if m != ref_m:     # n_dev_cases is sorted, so equal row counts are adjacent: one fp64 reference held at a time
            ref_m, ref = m, None
            ref = np_hash_bwd_f64(xnn[:m], dout[:m], lay, half, range(lay.levels))
        _check_scatter(N(g), prefill, *ref, 0, lay.total_param_size, f"n_dev={nd}")


# ---- B. generic feature width -----------------------------------------------------------------------------------------
GENERIC = {
    "deployment": (2 ** 21, 4, 32, 128, 4),   # the reference's --deployment model: all levels dense
    "hashed_f4": (2 ** 14, 8, 16, 1024, 4),
    "f1": (2 ** 16, 6, 16, 512, 1),
    "f3": (2 ** 16, 6, 16, 512, 3),
    "f8": (2 ** 16, 6, 16, 512, 8),
}
GENERIC_SCALE = {"deployment": 0.5}       # the box the _dyn variants normalise by (the Lego's for the deployment model)


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("F", [1, 3, 4, 8])
def test_oracle_generic_fwd_matches_numpy(oracle, F, half):
    """The GPU forward is compared bit for bit with the oracle, so the oracle's generic-F forward is held bit for bit
    to the independent numpy restatement, on hashed and dense levels, faces and corners."""
    from test_oracle import np_hash_encode
    rng = np.random.default_rng(50 + F + 10 * half)
    lay = make_hash_layout(2 ** 14, 6, 16, 512, F)
    assert 0 < lay.begin_fast_hash_level < lay.levels
    x = _unit_points(rng, 2000)
    table = rng.standard_normal(lay.total_param_size).astype(np.float32)
    table = (table * 0.1).astype(np.float16) if half else table
    with np.errstate(over="ignore"):
        ref = np_hash_encode(x, table, lay, half)
    got = oracle.hash_encode_fwd(x, table, lay)
    assert got.dtype == ref.dtype and got.shape == ref.shape
    view = np.uint16 if half else np.uint32
    assert np.array_equal(got.view(view), ref.view(view))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 63, 64, 65, 3000])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("name", list(GENERIC))
def test_hash_generic_fwd_bit_exact(lib, oracle, name, half, n):
    """One thread per (row, level) in blocks of 256: the n cover a partial block, a full one and one more row.  Rows
    past n keep the sentinel."""
    args = GENERIC[name]
    lay = _layout(args)
    cl = lay.as_ctypes()
    table = _table(args, half)
    x = _unit_points(np.random.default_rng(60 + n + half), n)
    ref = oracle.hash_encode_fwd(x, table, lay)
    dt, view = (torch.float16, np.uint16) if half else (torch.float32, np.uint32)
    out = torch.full((n + PAD, lay.out_dim), -7.0, device=DEV, dtype=dt)
    xs, tab = T(x), T(table)
    chk(lib.ngp_hash_encode_fwd(P(xs), P(tab), C.byref(cl), P(out), F16 if half else F32, n, ST()))
    got = N(out)
    assert np.array_equal(got[:n].view(view), ref.view(view)), "rows differ from the oracle"
    assert (got[n:] == -7.0).all(), "a row at or beyond n was written"


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("name", list(GENERIC))
def test_hash_generic_fwd_dyn_aabb_bit_exact(lib, oracle, name, half):
    """ngp_hash_encode_fwd_dyn with aabb6 and n_dev == the oracle on the fp32-normalised points, bit for bit, on the
    rows [0, min(n_max, max(n_dev, 0))); every other row keeps the sentinel."""
    args = GENERIC[name]
    scale = GENERIC_SCALE.get(name, 16.0)
    lay = _layout(args)
    cl = lay.as_ctypes()
    table = _table(args, half)
    n_max = 3000
    x = _world_points(np.random.default_rng(70 + half), n_max + PAD, scale)
    ref = oracle.hash_encode_fwd(_normalise(x[:n_max], scale), table, lay)
    dt, view = (torch.float16, np.uint16) if half else (torch.float32, np.uint32)
    xs, tab = T(x), T(table)
    for nd in n_dev_cases(n_max):
        out = torch.full((n_max + PAD, lay.out_dim), -7.0, device=DEV, dtype=dt)
        chk(lib.ngp_hash_encode_fwd_dyn(P(xs), P(tab), C.byref(cl), P(out), F16 if half else F32, n_max, P(i32(nd)),
                                        _aabb6(scale), ST()))
        got, m = N(out), rows_of(nd, n_max)
        assert np.array_equal(got[:m].view(view), ref[:m].view(view)), f"n_dev={nd}: rows differ from the oracle"
        assert (got[m:] == -7.0).all(), f"n_dev={nd}: a row at or beyond min(n_max, n_dev) was written"


def _generic_ray_points(rng, n, lay):
    """Ray samples one finest cell apart (where the F scalar atomics of neighbouring rows contend), with corner and
    face points."""
    return _on_faces(rng, _ray_points(rng, n, per_ray=200, step=1.0 / lay.max_res))


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("name", list(GENERIC))
def test_hash_generic_bwd_fp64_bound(lib, name, half):
    lay = _layout(GENERIC[name])
    cl = lay.as_ctypes()
    rng = np.random.default_rng(80 + half)
    n = 20000
    xn = _generic_ray_points(rng, n, lay)
    dout = _dout(rng, n, lay, half)
    _assert_dout_mix(dout, lay, n)
    xn = _poison_skipped_rows(rng, xn, dout, lay)
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    g, t_x, t_d = T(prefill), T(xn), T(dout)
    chk(lib.ngp_hash_encode_bwd(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n, ST()))
    ref, mag, cnt = np_hash_bwd_f64(xn, dout, lay, half, range(lay.levels))
    assert cnt.max() > 8   # contended entries
    _check_scatter(N(g), prefill, ref, mag, cnt, 0, lay.total_param_size, name)


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("name", list(GENERIC))
def test_hash_generic_bwd_dyn_aabb(lib, name, half):
    """World positions normalised inside the kernel and the row count read on the device: rows at or beyond
    min(n_max, n_dev) contribute nothing."""
    scale = GENERIC_SCALE.get(name, 16.0)
    lay = _layout(GENERIC[name])
    cl = lay.as_ctypes()
    rng = np.random.default_rng(90 + half)
    n_max = 3000
    xn = _generic_ray_points(rng, n_max + PAD, lay)
    dout = _dout(rng, n_max + PAD, lay, half)
    _assert_dout_mix(dout, lay, n_max // 2)
    xw = (xn * np.float32(2 * scale) - np.float32(scale)).astype(np.float32)
    xw[n_max // 2: n_max // 2 + n_max // 7] = _world_points(rng, n_max // 7, scale)
    xw = _poison_skipped_rows(rng, xw, dout, lay)
    xnn = _normalise(xw, scale)
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    t_x, t_d = T(xw), T(dout)
    ref_m = ref = None
    for nd in n_dev_cases(n_max):
        g = T(prefill)
        chk(lib.ngp_hash_encode_bwd_dyn(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n_max, P(i32(nd)),
                                        _aabb6(scale), ST()))
        m = rows_of(nd, n_max)
        if m != ref_m:     # equal row counts are adjacent (see test_hash_bwd_garden_dyn_aabb)
            ref_m, ref = m, None
            ref = np_hash_bwd_f64(xnn[:m], dout[:m], lay, half, range(lay.levels))
        _check_scatter(N(g), prefill, *ref, 0, lay.total_param_size, f"{name} n_dev={nd}")


# ---- C. input gradient --------------------------------------------------------------------------------------------------
DX_LAYOUTS = {1024: (2 ** 19, 16, 16, 1024, 2), 4096: GARDEN}


def _dx_inputs(max_res, half, n, seed):
    args = DX_LAYOUTS[max_res]
    lay = _layout(args)
    rng = np.random.default_rng(seed)
    x = _unit_points(rng, n)
    dout = rng.standard_normal((n, lay.out_dim)).astype(np.float32)
    return lay, x, _table(args, half), (dout.astype(np.float16) if half else dout)


def _check_dx(got, x, table, dout, lay, half, k, what):
    """|got - ref| <= k u sum |term| per component; at max_res 4096 in fp16 the inputs also separate the derivative
    of the forward (fraction p - f16(g)) from that of the fp32 forward (p - g) by more than the bound.  The reference
    is finite, so a non-finite component is outside the bound."""
    ref, mag = np_hash_dx_f64(x, table, dout, lay, half)
    assert np.isfinite(ref).all()
    err = np.abs(got.astype(np.float64) - ref)
    bad = np.flatnonzero((~(err <= k * U * mag)).any(1))
    assert bad.size == 0, (f"{what}: {bad.size} rows outside {k} u sum|term|, e.g. row {bad[0]} x {x[bad[0]]}: got "
                           f"{got[bad[0]]} ref {ref[bad[0]]} bound {k * U * mag[bad[0]]}")
    if half and lay.max_res > 2048 and len(x) > 1000:
        _assert_fp16_cast_exercised(x, lay)
        ref32, _ = np_hash_dx_f64(x, table, dout, lay, False)
        assert (np.abs(ref32 - ref) > k * U * mag).any()


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("max_res", [1024, 4096])
def test_oracle_dx_matches_fp64(oracle, max_res, half):
    lay, x, table, dout = _dx_inputs(max_res, half, 3000, 100 + max_res + half)
    _check_dx(oracle.hash_encode_bwd_input(x, table, dout, lay), x, table, dout, lay, half, 4, "oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 5000])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("max_res", [1024, 4096])
def test_hash_dx_fp64_bound(lib, max_res, half, n):
    """One thread per row in blocks of 256; rows past n keep the sentinel."""
    lay, x, table, dout = _dx_inputs(max_res, half, n, 110 + n + max_res + half)
    cl = lay.as_ctypes()
    dx = torch.full((n + PAD, 3), -7.0, device=DEV)
    t_x, t_t, t_d = T(x), T(table), T(dout)
    chk(lib.ngp_hash_encode_bwd_input(P(t_x), P(t_t), P(t_d), F16 if half else F32, C.byref(cl), P(dx), n, ST()))
    got = N(dx)
    assert (got[n:] == -7.0).all(), "a row at or beyond n was written"
    _check_dx(got[:n], x, table, dout, lay, half, 8 * lay.levels + 8, "kernel")


# ---- D. argument validation (CPU: rejected before any launch) ----------------------------------------------------
def test_hash_argument_validation_needs_no_gpu(lib):
    fake = C.c_void_p(0x10000)
    lay2 = _layout((2 ** 19, 16, 16, 1024, 2)).as_ctypes()
    fwd, fwd_dyn = lib.ngp_hash_encode_fwd, lib.ngp_hash_encode_fwd_dyn
    bwd, bwd_dyn, bwd_lv, bwd_x = (lib.ngp_hash_encode_bwd, lib.ngp_hash_encode_bwd_dyn,
                                   lib.ngp_hash_encode_bwd_levels, lib.ngp_hash_encode_bwd_input)
    for F in (1, 3, 4, 8):
        lay = make_hash_layout(2 ** 16, 6, 16, 512, F).as_ctypes()
        # dL/dx exists for F == 2 only
        assert bwd_x(fake, fake, fake, F32, C.byref(lay), fake, 8, None) < 0, F
        assert b"feature_per_level == 2" in lib.ngp_last_error()
        # a level group needs the F == 2 kernel
        for a, b in ((0, 3), (1, 6), (2, 3)):
            assert bwd_lv(fake, fake, F16, C.byref(lay), fake, 8, None, None, a, b, None, None) < 0, (F, a, b)
            assert b"level groups" in lib.ngp_last_error()
        # n = 0: a successful no-op, whatever the pointers
        assert fwd(None, None, C.byref(lay), None, F16, 0, None) == 0
        assert fwd_dyn(None, None, C.byref(lay), None, F32, 0, None, None, None) == 0
        assert bwd(None, None, F16, C.byref(lay), None, 0, None) == 0
        assert bwd_dyn(None, None, F32, C.byref(lay), None, 0, None, None, None) == 0
        assert bwd_x(None, None, None, F16, C.byref(lay), None, 0, None) == 0
    assert bwd_x(None, None, None, F32, C.byref(lay2), None, 0, None) == 0
    # widths outside [1, 8], level counts outside [1, 16], negative n, bad dtypes, null pointers
    for F in (0, 9):
        bad = make_hash_layout(2 ** 16, 6, 16, 512, 2).as_ctypes()
        bad.feat_dim = F
        assert fwd(fake, fake, C.byref(bad), fake, F32, 8, None) < 0
        assert b"feature_per_level" in lib.ngp_last_error()
        assert bwd(fake, fake, F32, C.byref(bad), fake, 8, None) < 0
    for L in (0, 17):
        bad = make_hash_layout(2 ** 16, 6, 16, 512, 2).as_ctypes()
        bad.n_levels = L
        assert fwd(fake, fake, C.byref(bad), fake, F32, 8, None) < 0
        assert b"n_levels" in lib.ngp_last_error()
    assert fwd(fake, fake, C.byref(lay2), fake, F32, -1, None) < 0
    assert bwd_x(fake, fake, fake, F32, C.byref(lay2), fake, -1, None) < 0
    assert fwd(fake, fake, C.byref(lay2), fake, 2, 8, None) < 0
    assert bwd(fake, fake, 2, C.byref(lay2), fake, 8, None) < 0
    assert bwd_x(fake, fake, fake, 2, C.byref(lay2), fake, 8, None) < 0
    assert fwd(fake, None, C.byref(lay2), fake, F32, 8, None) < 0
    assert bwd_x(fake, fake, None, F32, C.byref(lay2), fake, 8, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert fwd(fake, fake, None, fake, F32, 8, None) < 0
    # F = 2: the forward loads an x-pair of entries as one vector and the backward adds one as a 16-byte reduction, so
    # table must be aligned to two entries, grad_table to 16 bytes, out and dout to one entry
    at = lambda off: C.c_void_p(0x10000 + off)   # noqa: E731
    for dt, entry in ((F32, 8), (F16, 4)):
        for off in (entry, 2, 2 * entry + entry // 2):
            assert fwd(fake, at(off), C.byref(lay2), fake, dt, 8, None) < 0, (dt, off)
            assert b"table must be aligned to two entries" in lib.ngp_last_error()
            assert fwd_dyn(fake, at(off), C.byref(lay2), fake, dt, 8, None, None, None) < 0, (dt, off)
        for off in (entry // 2, entry + entry // 2):
            assert fwd(fake, fake, C.byref(lay2), at(off), dt, 8, None) < 0, (dt, off)
            assert b"out must be aligned to one entry" in lib.ngp_last_error()
            assert bwd(fake, at(off), dt, C.byref(lay2), fake, 8, None) < 0, (dt, off)
            assert b"dout must be aligned to one entry" in lib.ngp_last_error()
        assert bwd(fake, fake, dt, C.byref(lay2), at(8), 8, None) < 0
        assert b"grad_table must be 16-byte aligned" in lib.ngp_last_error()
        assert bwd_dyn(fake, fake, dt, C.byref(lay2), at(24), 8, None, None, None) < 0
        assert b"grad_table must be 16-byte aligned" in lib.ngp_last_error()
        for a, b in ((0, 16), (3, 7), (15, 16)):
            assert bwd_lv(fake, fake, dt, C.byref(lay2), at(8), 8, None, None, a, b, None, None) < 0, (a, b)
            assert b"grad_table must be 16-byte aligned" in lib.ngp_last_error()
        assert bwd(fake, fake, dt, C.byref(lay2), at(4), 8, None) < 0
        assert b"grad_table must be 8-byte aligned" in lib.ngp_last_error()
    # other widths keep their element-wise rule: grad_table 8-byte aligned
    lay4 = make_hash_layout(2 ** 16, 6, 16, 512, 4).as_ctypes()
    assert bwd(fake, fake, F32, C.byref(lay4), at(4), 8, None) < 0
    assert b"grad_table must be 8-byte aligned" in lib.ngp_last_error()
