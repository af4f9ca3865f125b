"""The tri-plane encoder kernels (csrc/triplane.cu) against fp64, per table float: the backward of both feature widths
(the F = 2 kernel scatters with red.global.add.v2.f32, the F = 4 kernel with .v4) under the scatter bound of
tests/triplane_ref.py, the forward bit-exact against the numpy restatement, on the same inputs.

Inputs: ray-coherent samples, points on every level's cell boundaries, the corners 0 and 1, and a slab of positions in
[-0.25, 1.25] that runs the max_res-grid clamp.  A fifth of the rows have dL/dout = 0 in some levels only (the kernel
skips those (row, level) pairs) and the gradient is prefilled, so accumulation is checked, not assignment.  The table
and the gradient sit in the middle of one allocation with half a plane of guard on each side: NaN in the table (an
out-of-table read poisons the forward), a sentinel in the gradient (an out-of-table write changes it).  Positions
never leave [-0.25, 1.25]: there even a kernel without the clamp reaches only a little more than a quarter plane past
the end, into the guard.  NaN, infinite and huge positions are not given to the GPU, where a wrong kernel could index
anywhere; the CPU oracle's clamp of those is tested by tests/test_triplane.py::test_oracle_forward_clamps_outside_unit_cube.

Also: max_res 16384 (every plane-2 float index >= 2^31), the device-counted forward with the folded AABB, and the
module's two gradient paths.  The CPU tests at the end feed the comparator the oracle's fp32 gradient and gradients
with the mistakes a looser check lets through.
"""
import numpy as np
import pytest

from hash_ref import PAD, _aabb6, _normalise, _ray_points, _world_points, n_dev_cases, rows_of
from taichi_nerfs_b200.layout import make_triplane_layout
from triplane_ref import (_check_triplane_scatter, _table_at, corner_entry, corner_weight, np_triplane_bwd_f64,
                          triplane_axes, triplane_numpy, triplane_ori)

DEV = "cuda"
SENTINEL = -1234.5


def T(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _slab(rng, n):
    return (rng.random((n, 3), dtype=np.float32) * np.float32(1.5) - np.float32(0.25)).astype(np.float32)


def _inputs(rng, lay):
    """Ray samples in [0, 1], test_gpu_triplane's cell-boundary / corner / slightly-outside points, a slab in
    [-0.25, 1.25]."""
    from test_gpu_triplane import _positions
    return np.concatenate([_ray_points(rng, 60000), _positions(rng, 20000, lay), _slab(rng, 20000)])


def _dout(rng, n, lay):
    """Normal dL/dout, column j*L + level; 20 % of the rows zero in a random proper subset of the levels, and single
    zero columns inside live levels (those rows still scatter: only an all-zero level is skipped)."""
    L, F = lay.levels, lay.feat_dim
    dy = rng.standard_normal((n, F, L)).astype(np.float32)
    zero = (rng.random(n) < 0.2)[:, None] & (rng.random((n, L)) < 0.5)
    zero[np.arange(n), rng.integers(0, L, n)] = False
    dy[np.broadcast_to(zero[:, None, :], dy.shape)] = 0.0
    dy[rng.random(dy.shape) < 0.05] = 0.0
    return dy.reshape(n, F * L)


def _prefill(rng, P):
    """Nonzero values of both signs, magnitude 2^-6 .. 3 * 2^-6."""
    p = rng.random(P, dtype=np.float32) + np.float32(0.5)
    p[1::2] *= np.float32(-1)
    return p * np.float32(1 / 32)


def _coverage(x, dout, lay):
    """Rows (among those a level of which scatters) with a clamped corner, with a level skipped by the zero-dy check
    while another scatters, and with two corners of one plane on the same entry."""
    n, L, F, mr = x.shape[0], lay.levels, lay.feat_dim, lay.max_res
    live = (dout.reshape(n, F, L) != 0).any(1)
    clamped, collide = np.zeros(n, bool), np.zeros(n, bool)
    for level in range(L):
        _, q = triplane_axes(x, lay, level)
        raw = [[triplane_ori(qb, mr, clamp=False) for qb in qk] for qk in q]
        ori = [[np.minimum(o, np.uint32(mr - 1)) for o in rk] for rk in raw]
        clamped |= live[:, level] & np.any([o > mr - 1 for rk in raw for o in rk], 0)
        collide |= live[:, level] & np.any([ok[0] == ok[1] for ok in ori], 0)
    return dict(rows=n, clamped=int(clamped.sum()), zero_dy=int(((~live).any(1) & live.any(1)).sum()),
                colliding=int(collide.sum()))


def _report(what, st):
    print(f"\n[{what}] {st}")


# ---- GPU: backward per float, forward bit-exact, guard bands --------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("levels,F,max_res", [(8, 4, 1024), (16, 2, 2048), (8, 2, 4096), (16, 4, 4096)])
def test_backward_per_float_fp64_and_forward_bit_exact(levels, F, max_res):
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(levels * 100 + F * 10 + max_res)
    lay = make_triplane_layout(levels, 16, max_res, F)
    assert lay.resolutions[-1] == max_res          # the finest level: grid lines 0 and 1 both map to max_res line 0
    cl = lay.as_ctypes()
    P, H = lay.total_param_size, max_res * max_res * F // 2
    x = _inputs(rng, lay)
    dout = _dout(rng, x.shape[0], lay)
    table = rng.random(P, dtype=np.float32)
    prefill = _prefill(rng, P)
    tab_all = torch.full((P + 2 * H,), float("nan"), device=DEV)
    grad_all = torch.full((P + 2 * H,), SENTINEL, device=DEV)
    tab, grad = tab_all[H:H + P], grad_all[H:H + P]
    tab.copy_(T(table))
    grad.copy_(T(prefill))
    xt = T(x)
    out = ops.triplane_encode_fwd(xt, tab, cl)
    ops.triplane_encode_bwd(xt, tab, T(dout), cl, grad)
    got = N(grad)
    guard = N(torch.cat([grad_all[:H], grad_all[H + P:]]))
    assert np.array_equal(guard.view(np.uint32), np.full(2 * H, SENTINEL, np.float32).view(np.uint32)), \
        "the backward wrote outside the table"
    assert torch.isnan(tab_all[:H]).all() and torch.isnan(tab_all[H + P:]).all()
    want = triplane_numpy(x, table, lay, clamp=True)
    assert np.array_equal(N(out).view(np.uint32), want.view(np.uint32)), "forward differs from the numpy restatement"
    idx, ref, mag, cnt = np_triplane_bwd_f64(x, _table_at(table), dout, lay)
    what = f"L={levels} F={F} max_res={max_res}"
    ratio = _check_triplane_scatter(got, prefill, idx, ref, mag, cnt, what)
    cov = _coverage(x, dout, lay)
    assert cov["clamped"] > 0 and cov["zero_dy"] > 0 and cov["colliding"] > 0, cov
    _report(what, dict(max_err_over_bound=ratio, floats_checked=int(idx.size), max_k=int(cnt.max()), **cov))


# ---- GPU: max_res 16384 ---------------------------------------------------------------------------------------------
HIGH_MASK = (1 << 20) - 1


def _high_table_at(e):
    """((e * 40503) mod 2^20) / 2^20 for float index e: exact in fp32."""
    return ((np.asarray(e, np.int64) * 40503) & HIGH_MASK).astype(np.float32) / np.float32(1 << 20)


def _fill_high_table(tab, chunk=1 << 27):
    import torch
    for s in range(0, tab.numel(), chunk):
        e = torch.arange(s, min(s + chunk, tab.numel()), device=DEV, dtype=torch.int64)
        tab[s:s + e.numel()] = ((e * 40503) & HIGH_MASK).float() / float(1 << 20)
        del e


def _count_nonzero(t, chunk=1 << 28):
    import torch
    return sum(int(torch.count_nonzero(t[s:s + chunk])) for s in range(0, t.numel(), chunk))


@pytest.mark.gpu
def test_max_res_16384_above_2_pow_31():
    """L=8, F=4, max_res 16384 (NGP_TRIPLANE_MAX_RES): table and gradient 12.9 GB each, every plane-2 float index
    >= 2^31, reached only through corner_entry's int64 arithmetic.  The table is a function of the float index, filled
    on the device; ~10^5 samples, half of them with z and x near 1 (the top of plane 2).  Forward bit-exact, backward
    within the fp64 bound on the touched floats, every other gradient float still zero."""
    import torch
    from taichi_nerfs_b200 import ops
    lay = make_triplane_layout(8, 16, 16384, 4)
    cl = lay.as_ctypes()
    P = lay.total_param_size
    assert 2 * 16384 ** 2 * 4 == 2 ** 31 and P * 4 > 12.8e9
    need = 2 * P * 4 + (6 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    rng = np.random.default_rng(16384)
    n = 100000
    x = rng.random((n, 3), dtype=np.float32)
    top = np.arange(n // 2, n)
    x[top, 0] = np.float32(1) - rng.random(top.size, dtype=np.float32) * np.float32(0.01)
    x[top, 2] = np.float32(1) - rng.random(top.size, dtype=np.float32) * np.float32(0.01)
    x[:4] = [[1, 1, 1], [0, 0, 0], [1, 0.5, 1], [0.999, 0.25, 1]]
    dout = _dout(rng, n, lay)
    torch.cuda.reset_peak_memory_stats()
    tab = grad = None
    try:
        tab = torch.empty(P, device=DEV)
        _fill_high_table(tab)
        grad = torch.zeros(P, device=DEV)
        xt = T(x)
        out = ops.triplane_encode_fwd(xt, tab, cl)
        ops.triplane_encode_bwd(xt, tab, T(dout), cl, grad)
        assert np.array_equal(N(out).view(np.uint32), triplane_numpy(x, _high_table_at, lay, clamp=True)
                              .view(np.uint32)), "forward differs from the numpy restatement"
        idx, ref, mag, cnt = np_triplane_bwd_f64(x, _high_table_at, dout, lay)
        assert (idx >= 2 ** 31).sum() > 0 and idx.max() >= P - 16384 * 4, "the top of plane 2 is not reached"
        it = T(idx)
        got = N(grad[it])
        ratio = _check_triplane_scatter(got, np.zeros_like(got), np.arange(idx.size), ref, mag, cnt, "max_res 16384")
        grad[it] = 0.0
        assert _count_nonzero(grad) == 0, "the backward wrote a float no sample reaches"
        peak = torch.cuda.max_memory_allocated()
        _report("L=8 F=4 max_res=16384", dict(max_err_over_bound=ratio, floats_checked=int(idx.size),
                                              above_2_31=int((idx >= 2 ** 31).sum()), max_k=int(cnt.max()),
                                              peak_gib=round(peak / 2 ** 30, 2)))
    finally:
        del tab, grad
        torch.cuda.empty_cache()


# ---- GPU: device row count with the folded AABB ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("scale", [0.5, 16.0])
@pytest.mark.parametrize("levels,F,max_res", [(8, 4, 1024), (16, 2, 2048)])
def test_forward_dyn_with_aabb(levels, F, max_res, scale):
    """ngp_triplane_encode_fwd_dyn with aabb6 and a device row count together (FrameRenderer's enqueue_encode_dyn):
    rows below min(n_max, max(n_dev, 0)) bit-exact against the numpy restatement of the fp32 normalisation
    (x - lo) / span, every row from there on, PAD included, untouched."""
    import ctypes as C

    import torch
    from taichi_nerfs_b200 import _lib, ops
    rng = np.random.default_rng(int(scale * 10) + F)
    lay = make_triplane_layout(levels, 16, max_res, F)
    cl = lay.as_ctypes()
    table = rng.random(lay.total_param_size, dtype=np.float32)
    n_max = 20000
    xw = _world_points(rng, n_max + PAD, scale)
    xn = _normalise(xw[:n_max], scale)
    assert (xn == 0).any() and (xn == 1).any()             # the box's faces and corners
    want = triplane_numpy(xn, table, lay, clamp=True)
    xt, tab = T(xw), T(table)
    lib = _lib.load()
    for nd in n_dev_cases(n_max):
        out = torch.full((n_max + PAD, lay.out_dim), -7.0, device=DEV)
        n_dev = torch.tensor([nd], device=DEV, dtype=torch.int32)
        _lib.check(lib.ngp_triplane_encode_fwd_dyn(ops._ptr(xt), ops._ptr(tab), C.byref(cl), ops._ptr(out), n_max,
                                                   ops._ptr(n_dev), _aabb6(scale), ops._stream()))
        got, m = N(out), rows_of(nd, n_max)
        assert np.array_equal(got[:m].view(np.uint32), want[:m].view(np.uint32)), f"n_dev={nd}: rows differ"
        assert (got[m:] == -7.0).all(), f"n_dev={nd}: a row at or beyond min(n_max, n_dev) was written"


# ---- GPU: the module's two gradient paths ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_module_default_encoder_gradients_fp64():
    """TriPlaneEncoder() (L=16, F=2, max_res 2048, the reference's default) through autograd: the returned
    plane_embedding.grad of one backward, then a grad_sink holding that gradient into which a second backward
    accumulates; both within the fp64 bound (k counts the contributions of both backwards)."""
    import torch
    from modules.triplane import TriPlaneEncoder
    from test_gpu_triplane import _positions
    torch.manual_seed(0)
    enc = TriPlaneEncoder().to(DEV)
    lay = enc._layout
    assert (lay.levels, lay.feat_dim, lay.max_res) == (16, 2, 2048)
    rng = np.random.default_rng(2048)
    x1 = _ray_points(rng, 60000)
    x2 = _positions(rng, 30000, lay)
    d1, d2 = _dout(rng, x1.shape[0], lay), _dout(rng, x2.shape[0], lay)
    table = N(enc.plane_embedding).copy()
    zeros = np.zeros(lay.total_param_size, np.float32)
    enc(T(x1)).backward(T(d1))
    g1 = enc.plane_embedding.grad
    r1 = _check_triplane_scatter(N(g1), zeros, *np_triplane_bwd_f64(x1, _table_at(table), d1, lay), "returned grad")
    sink = g1.detach().clone()
    enc.plane_embedding.grad = None
    enc.grad_sink = sink
    enc(T(x2)).backward(T(d2))
    assert enc.plane_embedding.grad is None
    ref2 = np_triplane_bwd_f64(np.concatenate([x1, x2]), _table_at(table), np.concatenate([d1, d2]), lay)
    r2 = _check_triplane_scatter(N(sink), zeros, *ref2, "grad_sink after two backwards")
    _report("TriPlaneEncoder()", dict(returned=r1, grad_sink=r2, floats_checked=int(ref2[0].size)))


# ---- CPU: the comparator accepts the oracle's gradient and rejects the mistakes -------------------------------------
FAULTS = ["plane_x1.001", "planes_0_1_swapped", "dlf0_from_lf0", "level_dropped", "columns_swapped",
          "ori_rounded", "unclamped"]


def _np_bwd_f32(x, table, dout, lay, grad, fault=None):
    """The backward in fp32 numpy, in the kernel's operation order (np.add.at: sequential atomics), with one planted
    mistake: dlf0 formed with lf0, a level dropped, the F columns of each scattered vector reversed, corner 1's
    max_res-grid coordinate rounded instead of truncated, or no clamp (reads clipped to the table, writes past its end
    dropped: what lands in the next plane stays there)."""
    n, L, F, mr = x.shape[0], lay.levels, lay.feat_dim, lay.max_res
    grad = grad.copy()
    cols = np.arange(F)
    for level in range(L):
        if fault == "level_dropped" and level == L - 1:
            continue
        dy = dout.reshape(n, F, L)[:, :, level]
        live = (dy != 0).any(1)
        xl, dy = x[live], dy[live]
        a, q = triplane_axes(xl, lay, level)
        ori = [[triplane_ori(qb, mr, clamp=fault != "unclamped") for qb in qk] for qk in q]
        if fault == "ori_rounded":
            ori = [[ok[0], np.minimum(np.rint(qk[1]).astype(np.uint32), np.uint32(mr - 1))] for ok, qk in zip(ori, q)]
        e = [[corner_entry(lay, ori, fd, c)[:, None] + cols for c in range(4)] for fd in range(3)]
        w = [[corner_weight(a, fd, c)[:, None] for c in range(4)] for fd in range(3)]
        lf = np.zeros((3, xl.shape[0], F), np.float32)
        for fd in range(3):
            for c in range(4):
                lf[fd] = lf[fd] + w[fd][c] * np.take(table, e[fd][c], mode="clip")
        d2 = dy * lf[2]
        dlf = [d2 * (lf[0] if fault == "dlf0_from_lf0" else lf[1]), d2 * lf[0], dy * (lf[0] * lf[1])]
        for fd in range(3):
            for c in range(4):
                g = w[fd][c] * dlf[fd]
                if fault == "columns_swapped":
                    g = g[:, ::-1]
                keep = e[fd][c] < grad.size
                np.add.at(grad, e[fd][c][keep], g[keep])
    return grad


@pytest.fixture(scope="module", params=[2, 4])
def cpu_case(request):
    from oracle import triplane as OT
    F = request.param
    rng = np.random.default_rng(F)
    lay = make_triplane_layout(4, 8, 64, F)
    x = np.concatenate([rng.random((2000, 3), dtype=np.float32), _slab(rng, 1000),
                        np.array([[0, 0, 0], [1, 1, 1], [0, 1, 0.5]], np.float32)])
    dout = _dout(rng, x.shape[0], lay)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    prefill = _prefill(rng, lay.total_param_size)
    ora = OT.triplane_encode_bwd(x, table, dout, lay, grad_table=prefill.copy())
    ref = np_triplane_bwd_f64(x, _table_at(table), dout, lay)
    return lay, x, dout, table, prefill, ora, ref


def test_comparator_accepts_the_oracle_and_numpy_gradients(cpu_case):
    lay, x, dout, table, prefill, ora, ref = cpu_case
    cov = _coverage(x, dout, lay)
    assert cov["clamped"] > 0 and cov["zero_dy"] > 0 and cov["colliding"] > 0, cov
    _check_triplane_scatter(ora, prefill, *ref, "oracle")
    _check_triplane_scatter(_np_bwd_f32(x, table, dout, lay, prefill), prefill, *ref, "numpy fp32")


@pytest.mark.parametrize("fault", FAULTS)
def test_comparator_rejects(cpu_case, fault):
    lay, x, dout, table, prefill, ora, ref = cpu_case
    plane = lay.total_param_size // 3
    delta = ora.astype(np.float64) - prefill
    if fault == "plane_x1.001":
        delta[plane:2 * plane] *= 1.001
        bad = (prefill + delta).astype(np.float32)
    elif fault == "planes_0_1_swapped":
        delta[:2 * plane] = np.concatenate([delta[plane:2 * plane], delta[:plane]])
        bad = (prefill + delta).astype(np.float32)
    else:
        bad = _np_bwd_f32(x, table, dout, lay, prefill, fault)
    assert not np.array_equal(bad, ora)
    with pytest.raises(AssertionError):
        _check_triplane_scatter(bad, prefill, *ref, fault)
