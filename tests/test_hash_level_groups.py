"""The level groups of the F = 2 hash-table backward (ngp_hash_bwd_level_groups): ngp_hash_encode_bwd_levels scatters
its level range one group per launch, each group's fp32 gradient slice at most half of the L2, so that the slice being
scattered stays resident.

- The plan for explicit L2 sizes (CPU): one group when the gradient fits, several when it does not, a level larger
  than the budget on its own; every level in exactly one group, groups contiguous, within budget and maximal.
- On the GPU, at the device's own L2 size and 2^20 rows (launches of fewer rows are never split): a level range that
  crosses a group boundary and one inside a group, against the fp64 scatter bound of tests/hash_ref.py.
"""
import ctypes as C

import numpy as np
import pytest

from taichi_nerfs_b200.layout import make_hash_layout

from hash_ref import _check_scatter, _level_slice, _ray_points, np_hash_bwd_f64

MIB = 1 << 20
F32, F16 = 0, 1


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def plan(lib, lay, a, b, l2_bytes):
    bounds = (C.c_int32 * 17)()
    g = lib.ngp_hash_bwd_level_groups(C.byref(lay.as_ctypes()), a, b, l2_bytes, bounds)
    assert g >= 1
    return list(bounds)[: g + 1]


def slice_bytes(lay, l):
    return lay.map_sizes[l] * lay.feat_dim * 4


def check_plan(lay, a, b, l2_bytes, bounds):
    assert bounds[0] == a and bounds[-1] == b
    assert all(x < y for x, y in zip(bounds, bounds[1:])), bounds     # contiguous, non-empty, each level once
    budget = l2_bytes // 2
    for g0, g1 in zip(bounds, bounds[1:]):
        size = sum(slice_bytes(lay, l) for l in range(g0, g1))
        assert size <= budget or g1 - g0 == 1, (bounds, g0, g1, size, budget)
        if g1 < b:                                                     # the next level would not have fitted
            assert size + slice_bytes(lay, g1) > budget, (bounds, g0, g1)


@pytest.mark.parametrize("max_res", [1024, 4096])
def test_plan_one_group_when_the_gradient_fits(lib, max_res):
    lay = make_hash_layout(2 ** 19, 16, 16, max_res, 2)
    total = lay.total_param_size * 4
    assert plan(lib, lay, 0, 16, 2 * total) == [0, 16]
    assert plan(lib, lay, 0, 16, 0) == [0, 16]                          # L2 size unknown: today's single launch


@pytest.mark.parametrize("max_res", [1024, 4096])
@pytest.mark.parametrize("l2_mib", [50, 40, 24])
@pytest.mark.parametrize("levels", [(0, 16), (3, 14), (6, 16)])
def test_plan_several_groups(lib, max_res, l2_mib, levels):
    lay = make_hash_layout(2 ** 19, 16, 16, max_res, 2)
    a, b = levels
    bounds = plan(lib, lay, a, b, l2_mib * MIB)
    check_plan(lay, a, b, l2_mib * MIB, bounds)
    if (a, b) == (0, 16):
        assert len(bounds) > 2


def test_plan_level_larger_than_the_budget(lib):
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)    # hashed levels: 4 MiB of gradient each
    l2 = 4 * MIB                                         # budget 2 MiB
    bounds = plan(lib, lay, 0, 16, l2)
    check_plan(lay, 0, 16, l2, bounds)
    fh = lay.begin_fast_hash_level
    assert bounds[-(16 - fh) - 1:] == list(range(fh, 17))   # every hashed level alone
    assert bounds[0] == 0 and bounds[1] <= fh


def test_plan_rejects_bad_arguments(lib):
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
    bounds = (C.c_int32 * 17)()
    cl = lay.as_ctypes()
    assert lib.ngp_hash_bwd_level_groups(C.byref(cl), 5, 5, 50 * MIB, bounds) < 0
    assert lib.ngp_hash_bwd_level_groups(C.byref(cl), 0, 17, 50 * MIB, bounds) < 0
    assert lib.ngp_hash_bwd_level_groups(C.byref(cl), 0, 16, 50 * MIB, None) < 0


# ---- the grouped scatter on the device ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("where", ["crosses_a_boundary", "inside_a_group"])
@pytest.mark.parametrize("half", [False, True])
def test_bwd_levels_grouped_fp64_bound(lib, half, where):
    import torch
    from taichi_nerfs_b200 import _lib
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    bounds = plan(lib, lay, 0, 16, l2)
    assert len(bounds) > 2, f"the full layout is one group at L2 = {l2} B: nothing to cross"
    if where == "crosses_a_boundary":       # levels 1 .. one past the first group: more than one budget
        a, b = 1, bounds[1] + 1
        assert len(plan(lib, lay, a, b, l2)) > 2
    else:
        g0, g1 = max(((x, y) for x, y in zip(bounds, bounds[1:])), key=lambda p: p[1] - p[0])
        a, b = (g0 + 1, g1) if g1 - g0 > 1 else (g0, g1)
        assert plan(lib, lay, a, b, l2) == [a, b]
    rng = np.random.default_rng(31 + half)
    n = 1 << 20                             # the smallest launch the backward splits into groups
    xn = _ray_points(rng, n)
    dout = rng.standard_normal((n, 32)).astype(np.float32)
    dout[rng.random(n) < 0.1] = 0.0
    dout = dout.astype(np.float16) if half else dout
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    dev = "cuda"
    g = torch.from_numpy(prefill).to(dev)
    t_x, t_d = torch.from_numpy(xn).to(dev), torch.from_numpy(dout).to(dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.ngp_hash_encode_bwd_levels(C.c_void_p(t_x.data_ptr()), C.c_void_p(t_d.data_ptr()),
                                              F16 if half else F32, C.byref(lay.as_ctypes()), C.c_void_p(g.data_ptr()),
                                              n, None, None, a, b, None, st))
    ref, mag, cnt = np_hash_bwd_f64(xn, dout, lay, half, range(a, b))
    lo, hi = _level_slice(lay, a, b)
    _check_scatter(g.cpu().numpy(), prefill, ref, mag, cnt, lo, hi, f"levels [{a},{b})")
