"""The five march entry points -- training count and write, the single-pass frame / graph-step march (with and without
jitter), the compacting renderer's round march and the module test loop's march -- on the rays at the edges of the
march (tests/march_ref.py: axis-parallel directions with +-0 components, origins on cell and AABB faces, rays through
the exact origin, grazing rays, constant-dt chains whose binade boundary falls at chunk lanes 0, 1, 15, 31 and 32,
direction components at the -1e-3 threshold of the warp march's regular path) and on rays the reference never ends.
Every output is compared bit for bit with the CPU oracle and passes the fp64 checks of march_ref.check_samples."""
import ctypes as C

import numpy as np
import pytest
import torch

import march_ref as R

pytestmark = pytest.mark.gpu

f32 = np.float32
G = 128
DEV = "cuda"

# (scale, cascades, exp_step_factor, occupancy)
EDGE_CFGS = {
    "scale0.5_random": (0.5, 1, 0.0, "random"),
    "scale0.5_full": (0.5, 1, 0.0, "full"),            # every position emitted: the chunk chain itself is compared
    "5casc_scale8": (8.0, 5, 1 / 256, "random"),
    "5casc_scale8_full": (8.0, 5, 1 / 256, "full"),     # long chords: rays reach max_samples = 1024
    "3casc_scale1.5": (1.5, 3, 1 / 256, "sparse"),
}


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def _same(a, b, nan=False):
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    if nan:   # NaN payloads differ between the host and the device; positions of a NaN ray compare as NaN
        return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.fixture(scope="module")
def ops():
    from taichi_nerfs_b200 import ops as o
    return o


def _bits(occ, casc, rng):
    nbytes = casc * G ** 3 // 8
    if occ == "full":
        return np.full(nbytes, 255, np.uint8)
    if occ == "empty":
        return np.zeros(nbytes, np.uint8)
    if occ == "random":
        return rng.integers(0, 256, nbytes, dtype=np.uint8)
    return (rng.random(nbytes) < 0.05).astype(np.uint8) * rng.integers(1, 256, nbytes, dtype=np.uint8)


def _inputs(name, rays_factory, seed=50):
    scale, casc, esf, occ = EDGE_CFGS[name]
    rng = np.random.default_rng(seed)
    o, d = rays_factory(1000, seed=seed, radius=1.4 if scale == 0.5 else 3.0)
    eo, ed, eh, names = R.edge_rays(scale, seed=seed)
    hits = np.concatenate([R.aabb(o, d, scale), eh])
    return np.concatenate([o, eo]), np.concatenate([d, ed]), hits, _bits(occ, casc, rng), rng


def _rows(ra):
    """rays_a [m, 3] -> (ray of every row, row index), rows listed slot by slot."""
    k = ra[:, 2].astype(np.int64)
    off = np.repeat(ra[:, 1].astype(np.int64) - (np.cumsum(k) - k), k)
    return np.repeat(ra[:, 0], k), off + np.arange(int(k.sum()))


def _train(ops, o, d, hits, bits, noise, casc, sc, esf, m):
    counter, rays_a = ops.raymarching_train_count(T(o), T(d), T(hits), T(bits), T(noise), casc, sc, esf, G, m)
    S = int(counter[0])
    bufs = [torch.zeros(S, 3, device=DEV), torch.zeros(S, 3, device=DEV), torch.zeros(S, device=DEV),
            torch.zeros(S, device=DEV)]
    ops.raymarching_train_write(T(o), T(d), T(hits), T(bits), T(noise), casc, sc, esf, G, counter, rays_a, *bufs)
    ra = N(rays_a)
    ray, idx = _rows(ra)
    x, _, dl, t = (N(b) for b in bufs)
    return ra[:, 2], ray, t[idx], dl[idx], x[idx]


def _frame(ops, o, d, hits, bits, noise, casc, sc, esf, m, cap):
    n = o.shape[0]
    counter = torch.zeros(2, device=DEV, dtype=torch.int32)
    rays_a = torch.zeros(n, 3, device=DEV, dtype=torch.int32)
    bufs = [torch.zeros(cap, 3, device=DEV), torch.zeros(cap, 3, device=DEV), torch.zeros(cap, device=DEV),
            torch.zeros(cap, device=DEV)]
    ops.raymarching_frame(T(o), T(d), T(hits), T(bits), casc, sc, esf, G, m, counter, rays_a, *bufs,
                          noise=None if noise is None else T(noise))
    assert int(counter[1]) == 0                                     # nothing dropped for lack of capacity
    ra = N(rays_a)
    order = np.argsort(ra[:, 0], kind="stable")
    ray, idx = _rows(ra[order])
    x, _, dl, t = (N(b) for b in bufs)
    cnt = np.zeros(n, np.int64)
    cnt[ra[:, 0]] = ra[:, 2]
    return cnt, ray, t[idx], dl[idx], x[idx]


def _round(o, d, hits, bits, casc, sc, esf, m):
    """The compacting renderer's round march, every ray on the live list each round, with a changing per-round limit
    until every ray has left the box or reached m samples; rows regrouped by ray."""
    from taichi_nerfs_b200 import _lib
    L = _lib.load()
    n = o.shape[0]
    to, td, tb, th = T(o), T(d), T(bits), T(hits)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    cap = 64 * n
    t_cur = torch.where(th[:, 0] > 0, th[:, 0], torch.full_like(th[:, 0], -1.0)).contiguous()
    n_marched = torch.zeros(n, device=DEV, dtype=torch.int32)
    alive = torch.arange(n, device=DEV, dtype=torch.int32)
    state = torch.zeros(8, device=DEV, dtype=torch.int32)
    r_a = torch.zeros(n, 3, device=DEV, dtype=torch.int32)
    xyz, dirs = torch.empty(cap, 3, device=DEV), torch.empty(cap, 3, device=DEV)
    dl, ts = torch.empty(cap, device=DEV), torch.empty(cap, device=DEV)
    rows = ([], [], [], [])
    schedule = [1, 31, 4, 33, 64, 512]
    for k in range(64):
        if bool(((t_cur == float("inf")) | (t_cur < 0)).all()):
            break
        state.zero_()
        state[2] = n
        _lib.check(L.ngp_raymarching_round(p(to), p(td), p(th), p(tb), casc, G, sc, esf, schedule[min(k, 5)], m,
                                           p(alive), p(state), p(t_cur), p(n_marched), p(r_a), p(xyz), p(dirs), p(dl),
                                           p(ts), n, cap, st))
        ray, idx = _rows(N(r_a))
        for lst, a in zip(rows, (ray, N(ts)[idx], N(dl)[idx], N(xyz)[idx])):
            lst.append(a)
    assert bool(((t_cur == float("inf")) | (t_cur < 0)).all()), "every ray must end"
    ray = np.concatenate(rows[0])
    order = np.argsort(ray, kind="stable")
    return (N(n_marched), ray[order]) + tuple(np.concatenate(r)[order] for r in rows[1:])


def _test_march(ops, o, d, hits, bits, alive, casc, sc, esf, m):
    A = alive.shape[0]
    h = T(hits)
    g_ri = torch.zeros(A * m, device=DEV, dtype=torch.long)
    g_valid = torch.zeros(A * m, device=DEV, dtype=torch.uint8)
    g_dl, g_tt = torch.zeros(A * m, device=DEV), torch.zeros(A * m, device=DEV)
    g_cnt = torch.zeros(A, device=DEV, dtype=torch.int32)
    ops.raymarching_test(T(o), T(d), h, T(alive), T(bits), casc, sc, esf, G, m, g_ri, g_valid, g_dl, g_tt, g_cnt)
    return N(g_cnt), N(g_valid), N(g_ri), N(g_dl), N(g_tt), N(h)


@pytest.mark.parametrize("max_samples", [1, 31, 33, 1024])
@pytest.mark.parametrize("name", list(EDGE_CFGS))
def test_march_entry_points_on_edge_rays(ops, oracle, rays_factory, name, max_samples):
    sc, casc, esf, occ = EDGE_CFGS[name]
    o, d, hits, bits, rng = _inputs(name, rays_factory)
    n, m = o.shape[0], max_samples
    assert _same(N(ops.ray_aabb_intersect(T(o), T(d), sc)), oracle.ray_aabb_intersect(o, d, sc))
    noise = rng.random(n, dtype=f32)
    zero = np.zeros(n, f32)
    want = {}
    for key, nz in (("jitter", noise), ("zero", zero)):
        ra, xyzs, _, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, nz, casc, sc, esf, G, m)
        want[key] = (ra[:, 2], np.repeat(ra[:, 0], ra[:, 2]), ts, deltas, xyzs)
    if m == 1024 and occ == "full" and sc > 0.5:
        assert (want["zero"][0] == 1024).any()                      # the single-pass buffer fills up
    cap = max(int(w[0].sum()) for w in want.values()) + 100
    got = {
        "train count/write": (_train(ops, o, d, hits, bits, noise, casc, sc, esf, m), "jitter"),
        "frame, graph step": (_frame(ops, o, d, hits, bits, noise, casc, sc, esf, m, cap), "jitter"),
        "frame, test time": (_frame(ops, o, d, hits, bits, None, casc, sc, esf, m, cap), "zero"),
        "round march": (_round(o, d, hits, bits, casc, sc, esf, m), "zero"),
    }
    for what, (g, key) in got.items():
        w = want[key]
        assert np.array_equal(g[0], w[0]), what
        assert np.array_equal(g[1], w[1]), what
        for a, b in zip(g[2:], w[2:]):
            assert _same(a, b), what
        R.check_samples(o, d, hits, g[1], g[2], g[3], g[4], bits, casc, sc, esf)
    # the module test loop's march, resume points included
    alive = np.arange(n, dtype=np.int64)
    mt = min(m, 64)
    h_ref = hits.copy()
    ri, valid, dl, tt, cnt = oracle.raymarching_test(o, d, h_ref, alive, bits, casc, sc, esf, G, mt)
    g_cnt, g_valid, g_ri, g_dl, g_tt, g_h = _test_march(ops, o, d, hits, bits, alive, casc, sc, esf, mt)
    assert np.array_equal(g_cnt, cnt) and np.array_equal(g_valid, valid)
    v = valid.astype(bool)
    assert np.array_equal(g_ri[v], ri[v]) and _same(g_dl[v], dl[v]) and _same(g_tt[v], tt[v])
    assert _same(g_h, h_ref)
    x = (o[g_ri[v]] + g_tt[v][:, None] * d[g_ri[v]]).astype(f32)
    R.check_samples(o, d, hits, g_ri[v], g_tt[v], g_dl[v], x, bits, casc, sc, esf)


@pytest.mark.parametrize("occ", ["empty", "full"])
@pytest.mark.parametrize("sc,casc,esf", [(0.5, 1, 0.0), (8.0, 5, 1 / 256)])
def test_march_entry_points_end_degenerate_rays(ops, oracle, sc, casc, esf, occ):
    """Zero and NaN directions, a NaN origin, direction 1e-30: the reference never ends these rays.  The AABB kernel
    reports a miss where the far hit is not finite; every march entry point, given the reference's intervals
    [0.01, +inf) and [0.01, 2e29), ends each ray -- with no sample in an empty grid, with at most max_samples in a
    full one -- and agrees with the oracle."""
    o, d, _ = R.degenerate_rays()
    n = o.shape[0]
    got_hits = N(ops.ray_aabb_intersect(T(o), T(d), sc))
    assert _same(got_hits, oracle.ray_aabb_intersect(o, d, sc))
    assert (got_hits[:3] == -1).all() and np.isfinite(got_hits[3]).all()
    hits = np.array([[0.01, np.inf]] * 3 + [[0.01, got_hits[3, 1]]], f32)
    bits = _bits(occ, casc, None)
    zero = np.zeros(n, f32)
    ra, xyzs, _, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, zero, casc, sc, esf, G, 1024)
    if occ == "empty":
        assert S == 0
    want = (ra[:, 2], np.repeat(ra[:, 0], ra[:, 2]), ts, deltas, xyzs)
    for what, g in (("train count/write", _train(ops, o, d, hits, bits, zero, casc, sc, esf, 1024)),
                    ("frame, graph step", _frame(ops, o, d, hits, bits, zero, casc, sc, esf, 1024, S + 100)),
                    ("frame, test time", _frame(ops, o, d, hits, bits, None, casc, sc, esf, 1024, S + 100)),
                    ("round march", _round(o, d, hits, bits, casc, sc, esf, 1024))):
        assert np.array_equal(g[0], want[0]) and np.array_equal(g[1], want[1]), what
        assert _same(g[2], want[2]) and _same(g[3], want[3]) and _same(g[4], want[4], nan=True), what
    alive = np.arange(n, dtype=np.int64)
    h_ref = hits.copy()
    ri, valid, dl, tt, cnt = oracle.raymarching_test(o, d, h_ref, alive, bits, casc, sc, esf, G, 64)
    g_cnt, g_valid, g_ri, g_dl, g_tt, g_h = _test_march(ops, o, d, hits, bits, alive, casc, sc, esf, 64)
    assert np.array_equal(g_cnt, cnt) and np.array_equal(g_valid, valid)
    v = valid.astype(bool)
    assert _same(g_dl[v], dl[v]) and _same(g_tt[v], tt[v]) and _same(g_h, h_ref)
