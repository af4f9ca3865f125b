"""GPU parity: every CUDA kernel (called through the C-ABI via taichi_nerfs_b200.ops) against the CPU
oracle on the same seeded inputs.  Integer/index work and marching are compared bit-exactly; fp paths
within the tolerance stated next to each assert (north_star: 1e-3 relative for fp16 paths)."""
import numpy as np
import pytest
import torch

from taichi_nerfs_b200.layout import make_hash_layout

pytestmark = pytest.mark.gpu

DEV = "cuda"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def ops():
    from taichi_nerfs_b200 import ops as o
    return o


# ---- a1 -------------------------------------------------------------------------------------------
def test_ray_aabb_bit_exact(ops, oracle, rays_factory):
    o, d = rays_factory(10007, seed=20)
    d[:50] *= -1
    d[50:60, 0] = 0.0  # axis-parallel rays (division by zero -> inf, still IEEE)
    ref = oracle.ray_aabb_intersect(o, d, 0.5)
    got = N(ops.ray_aabb_intersect(T(o), T(d), 0.5))
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


# ---- a2 -------------------------------------------------------------------------------------------
MARCH_CFGS = [
    dict(scale=0.5, cascades=1, esf=0.0, occ="lego"),
    dict(scale=0.5, cascades=1, esf=0.0, occ="random"),
    dict(scale=16.0, cascades=6, esf=1 / 256, occ="random"),
    dict(scale=2.0, cascades=3, esf=1 / 256, occ="sparse"),
    dict(scale=8.0, cascades=5, esf=1 / 256, occ="random"),     # the scale README.md ships for real scenes
    dict(scale=1.5, cascades=3, esf=1 / 256, occ="random"),     # top cascade bound 1.5 (not a power of two)
    dict(scale=3.0, cascades=4, esf=1 / 256, occ="sparse"),     # top cascade bound 3
    dict(scale=64.0, cascades=8, esf=1 / 256, occ="random"),
]
MARCH_IDS = ["lego", "random", "6casc_esf", "3casc_sparse", "5casc_scale8", "3casc_scale1.5", "4casc_scale3",
             "8casc_scale64"]


def _march_inputs(cfg, n, seed, rng, rays_factory, lego_bitfield):
    """Rays (inside the box unless the scene is the Lego one) and an occupancy bitfield of one march configuration."""
    radius = 1.4 if cfg["scale"] == 0.5 else 3.0
    o, d = rays_factory(n, seed=seed, radius=radius)
    nbytes = cfg["cascades"] * 128 ** 3 // 8
    if cfg["occ"] == "lego":
        bits = lego_bitfield
    elif cfg["occ"] == "full":
        bits = np.full(nbytes, 255, np.uint8)
    elif cfg["occ"] == "random":
        bits = rng.integers(0, 256, nbytes, dtype=np.uint8)
    else:
        bits = (rng.random(nbytes) < 0.02).astype(np.uint8) * rng.integers(1, 256, nbytes, dtype=np.uint8)
    return o, d, bits


def _row_order(ra):
    """rays_a [m, 3] -> (ray of every row, row index), rows listed slot by slot."""
    k = ra[:, 2].astype(np.int64)
    off = np.repeat(ra[:, 1].astype(np.int64) - (np.cumsum(k) - k), k)
    return np.repeat(ra[:, 0], k), off + np.arange(int(k.sum()))


@pytest.mark.parametrize("cfg", MARCH_CFGS)
def test_march_train_bit_exact(ops, oracle, rays_factory, lego_bitfield, cfg):
    n = 4099
    rng = np.random.default_rng(21)
    o, d, bits = _march_inputs(cfg, n, 21, rng, rays_factory, lego_bitfield)
    hits = oracle.ray_aabb_intersect(o, d, cfg["scale"])
    noise = rng.random(n, dtype=np.float32)
    ra, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, noise, cfg["cascades"], cfg["scale"],
                                                            cfg["esf"], 128, 1024)
    from modules.ray_march import raymarching_train
    g_ra, g_xyzs, g_dirs, g_deltas, g_ts, g_total = raymarching_train(
        T(o), T(d), T(hits), T(bits), cfg["cascades"], cfg["scale"], cfg["esf"], 128, 1024, noise=T(noise))
    assert int(g_total) == S
    assert np.array_equal(N(g_ra), ra)
    for a, b in ((g_xyzs, xyzs), (g_dirs, dirs), (g_deltas, deltas), (g_ts, ts)):
        assert np.array_equal(N(a).view(np.uint32), b.view(np.uint32))


def test_march_train_empty_and_overflow(ops, oracle, rays_factory, lego_bitfield):
    n = 512
    o, d = rays_factory(n, seed=22)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = np.zeros(n, np.float32)
    # empty grid -> zero samples
    empty = np.zeros_like(lego_bitfield)
    counter, rays_a = ops.raymarching_train_count(T(o), T(d), T(hits), T(empty), T(noise), 1, 0.5, 0.0, 128, 1024)
    assert N(counter).tolist() == [0, n] and not N(rays_a)[:, 2].any()
    # capacity smaller than the total: rays that do not fit are dropped as a suffix
    ra, *_, S = oracle.raymarching_train(o, d, hits, lego_bitfield, noise, 1, 0.5, 0.0, 128, 1024)
    cap = S // 2
    tb = T(lego_bitfield)
    counter, rays_a = ops.raymarching_train_count(T(o), T(d), T(hits), tb, T(noise), 1, 0.5, 0.0, 128, 1024)
    bufs = [torch.zeros(cap, 3, device=DEV), torch.zeros(cap, 3, device=DEV), torch.zeros(cap, device=DEV),
            torch.zeros(cap, device=DEV)]
    ops.raymarching_train_write(T(o), T(d), T(hits), tb, T(noise), 1, 0.5, 0.0, 128, counter, rays_a, *bufs)
    c = N(counter)
    g = N(rays_a)
    assert c[0] <= cap and c[0] == g[:, 2].sum()
    kept = g[:, 2] > 0
    assert np.array_equal(g[kept, 2], ra[kept, 2])
    dropped = (~kept) & (ra[:, 2] > 0)
    assert dropped.any()
    assert not kept[np.argmax(dropped):].any()  # dropped rays form a suffix


# ---- a3 -------------------------------------------------------------------------------------------
# the Lego configuration keeps its ids (the max_samples alone); every other configuration at two chunk sizes
MARCH_TEST_CASES = [pytest.param(MARCH_CFGS[0], m, id=str(m)) for m in (1, 4, 64)] + [
    pytest.param(c, m, id=f"{i}-{m}") for c, i in zip(MARCH_CFGS[1:], MARCH_IDS[1:]) for m in (4, 64)]


@pytest.mark.parametrize("cfg,max_samples", MARCH_TEST_CASES)
def test_march_test_bit_exact(ops, oracle, rays_factory, lego_bitfield, cfg, max_samples):
    n = 3001
    o, d, bits = _march_inputs(cfg, n, 23, np.random.default_rng(23), rays_factory, lego_bitfield)
    sc, casc, esf = cfg["scale"], cfg["cascades"], cfg["esf"]
    hits = oracle.ray_aabb_intersect(o, d, sc)
    alive = np.random.default_rng(23).permutation(n)[: n // 2].astype(np.int64)
    h_ref = hits.copy()
    ri, valid, dl, tt, cnt = oracle.raymarching_test(o, d, h_ref, alive, bits, casc, sc, esf, 128, max_samples)
    h_gpu = T(hits)
    A, m = alive.shape[0], max_samples
    g_ri = torch.zeros(A * m, device=DEV, dtype=torch.long)
    g_valid = torch.zeros(A * m, device=DEV, dtype=torch.uint8)
    g_dl = torch.zeros(A * m, device=DEV)
    g_tt = torch.zeros(A * m, device=DEV)
    g_cnt = torch.zeros(A, device=DEV, dtype=torch.int32)
    ops.raymarching_test(T(o), T(d), h_gpu, T(alive), T(bits), casc, sc, esf, 128, m, g_ri, g_valid, g_dl, g_tt, g_cnt)
    assert np.array_equal(N(g_cnt), cnt)
    assert np.array_equal(N(g_valid), valid)
    v = valid.astype(bool)
    assert np.array_equal(N(g_ri)[v], ri[v])
    assert np.array_equal(N(g_dl)[v].view(np.uint32), dl[v].view(np.uint32))
    assert np.array_equal(N(g_tt)[v].view(np.uint32), tt[v].view(np.uint32))
    assert np.array_equal(N(h_gpu).view(np.uint32), h_ref.view(np.uint32))  # in-place resume points


# ---- a4/a5 ----------------------------------------------------------------------------------------
def _table(rng, lay, half):
    if half:
        return ((rng.random(lay.total_param_size, dtype=np.float32) * 2 - 1) * 1e-4).astype(np.float16)
    return rng.random(lay.total_param_size, dtype=np.float32)


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("max_res", [1024, 4096])
@pytest.mark.parametrize("n", [1, 127, 5000])
def test_hash_fwd_bit_exact(ops, oracle, half, max_res, n):
    rng = np.random.default_rng(24)
    lay = make_hash_layout(2 ** 19, 16, 16, max_res, 2)
    xyz = rng.random((n, 3), dtype=np.float32)
    xyz[: min(n, 4)] = np.array([[0, 0, 0], [1, 1, 1], [0, 1, 0.5], [1, 0, 1]], np.float32)[: min(n, 4)]
    table = _table(rng, lay, half)
    ref = oracle.hash_encode_fwd(xyz, table, lay)
    got = N(ops.hash_encode_fwd(T(xyz), T(table), lay.as_ctypes(), lay.out_dim))
    assert got.dtype == ref.dtype and got.shape == ref.shape
    # identical op order on both sides (no FMA contraction) -> bit exact, fp16 and fp32
    assert np.array_equal(got.view(np.uint8), ref.view(np.uint8))


@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_matches_oracle(ops, oracle, half):
    rng = np.random.default_rng(25)
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
    n = 20000
    # samples along rays: spatially coherent like real marching output (stresses atomic contention)
    base = rng.random((n // 100, 1, 3), dtype=np.float32) * 0.8 + 0.1
    xyz = (base + (np.arange(100, dtype=np.float32)[None, :, None] * 0.0015)).reshape(-1, 3).clip(0, 1).astype(np.float32)
    dout = rng.standard_normal((n, 32)).astype(np.float32)
    dout[rng.random(n) < 0.1] = 0.0  # zero-gradient samples are skipped (hash_encoder_half.py:210)
    if half:
        dout = dout.astype(np.float16)
    ref = oracle.hash_encode_bwd(xyz, dout, lay)
    g = torch.zeros(lay.total_param_size, device=DEV)
    ops.hash_encode_bwd(T(xyz), T(dout), lay.as_ctypes(), g)
    got = N(g)
    # fp32 atomics in arbitrary order vs sequential fp32 sums: 1e-3 relative (north_star tolerance)
    # measured against the per-level gradient magnitude
    assert np.array_equal(got == 0, ref == 0)
    np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-3 * np.abs(ref).max() * 1e-2)


def test_hash_bwd_input_matches_oracle(ops, oracle):
    rng = np.random.default_rng(26)
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
    n = 3000
    xyz = rng.random((n, 3), dtype=np.float32)
    table = rng.standard_normal(lay.total_param_size).astype(np.float32)
    dout = rng.standard_normal((n, 32)).astype(np.float32)
    ref = oracle.hash_encode_bwd_input(xyz, table, dout, lay)
    got = N(ops.hash_encode_bwd_input(T(xyz), T(table), T(dout), lay.as_ctypes()))
    np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-3 * np.abs(ref).max())


def test_hash_autograd_modules(oracle):
    """HashEncoder drop-in modules: forward + backward through torch.autograd."""
    from modules.hash_encoder import HashEncoder as H32
    from modules.hash_encoder_half import HashEncoder as H16
    rng = np.random.default_rng(27)
    x = rng.random((4000, 3), dtype=np.float32)
    for cls, half in ((H32, False), (H16, True)):
        enc = cls(max_params=2 ** 19, levels=16, base_res=16, max_res=1024).to(DEV)
        lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
        out = enc(T(x))
        tab = N(enc.hash_table).reshape(-1)
        ref = oracle.hash_encode_fwd(x, tab.astype(np.float16) if half else tab, lay)
        assert np.array_equal(N(out).view(np.uint8), ref.view(np.uint8))
        dout = rng.standard_normal(ref.shape).astype(ref.dtype)
        out.backward(T(dout))
        gref = oracle.hash_encode_bwd(x, dout, lay)
        np.testing.assert_allclose(N(enc.hash_table.grad).reshape(-1), gref, rtol=1e-3, atol=1e-5)
        assert enc.hash_table.grad.shape == enc.hash_table.shape


# ---- a6 -------------------------------------------------------------------------------------------
def test_dir_encode(ops, oracle):
    rng = np.random.default_rng(28)
    d = rng.random((5003, 3), dtype=np.float32)
    ref = oracle.dir_encode(d)
    got = N(ops.dir_encode(T(d)))
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-7)  # nvcc may contract a*b+c into fma


# ---- a7 -------------------------------------------------------------------------------------------
def _weights(rng):
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    return [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]


@pytest.mark.parametrize("emb_half", [True, False])
@pytest.mark.parametrize("n", [1, 128, 1000, 70001])
def test_mlp_fwd_tcgen05_matches_oracle(ops, oracle, emb_half, n):
    _mlp_fwd_matches_oracle(ops, oracle, emb_half, n, "xavier")


@pytest.mark.parametrize("emb_half", [True, False])
@pytest.mark.parametrize("n", [1, 128, 1000, 70001])
def test_mlp_fwd_tcgen05_matches_oracle_trained(ops, oracle, emb_half, n):
    """The same comparison on the finite regimes of tests/mlp_tolerance.py::trained_inputs (h0 beyond and within an
    ulp16 of +-15, |h0| in 8..11, fp16 sigmoid exactly 0 / 1) at the first / last row and on 64-row tile edges."""
    _mlp_fwd_matches_oracle(ops, oracle, emb_half, n, "trained")


def _mlp_fwd_matches_oracle(ops, oracle, emb_half, n, magnitude):
    rng = np.random.default_rng(29)
    emb = rng.standard_normal((n, 32)).astype(np.float16 if emb_half else np.float32)
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    ws = _weights(rng)
    if magnitude == "trained":
        from mlp_tolerance import trained_inputs
        emb, dirs, ws, _, _, _ = trained_inputs(n, 29, np.float16 if emb_half else np.float32)
    sig_ref, rgb_ref = oracle.mlp_fwd(emb, dirs, ws)
    sig, rgb = ops.mlp_fwd(T(emb), T(dirs), [T(w) for w in ws])
    sig, rgb = N(sig), N(rgb).astype(np.float32)
    # per-element fp16 flip model (tests/mlp_tolerance.py): rigorous bound on every element, 99 % of the elements
    # within 2 ulp16(h0) (= 1e-3 relative on sigma for |h0| < 1), median exact; rgb in [0,1]: 4 fp16 ulp absolute
    from mlp_tolerance import check_sigma
    check_sigma(sig, sig_ref, emb, ws)
    assert np.abs(rgb - rgb_ref.astype(np.float32)).max() <= 2e-3
    assert np.median(np.abs(sig - sig_ref) / sig_ref) < 1e-3


# ---- a8 -------------------------------------------------------------------------------------------
def _composite_inputs(rng, n_rays, max_n, dense, half):
    counts = rng.integers(0, max_n, n_rays)
    counts[:3] = [0, 1, 33]
    S = int(counts.sum())
    rays_a = np.stack([rng.permutation(n_rays), np.cumsum(counts) - counts, counts], 1).astype(np.int32)
    sig = (rng.random(S) * (60.0 if dense else 3.0)).astype(np.float32)
    rgbs = rng.random((S, 3)).astype(np.float16 if half else np.float32)
    deltas = np.full(S, 1.7320508075688772 / 1024 * (20 if dense else 1), np.float32)
    ts = np.sort(rng.random(S)).astype(np.float32)
    return rays_a, sig, rgbs, deltas, ts


@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("half", [False, True])
def test_composite_train_fwd_bwd(ops, oracle, dense, half):
    rng = np.random.default_rng(30)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, 700, 300, dense, half)
    n, S = rays_a.shape[0], sig.shape[0]
    tot, op, dep, rgb, ws = oracle.composite_train_fwd(sig, rgbs, deltas, ts, rays_a, 1e-4)
    g = ops.composite_train_fwd(T(sig), T(rgbs), T(deltas), T(ts), T(rays_a), 1e-4)
    g_tot, g_op, g_dep, g_rgb, g_ws = [N(x) for x in g]
    # warp prefix products vs sequential products: 1e-5 absolute on O(1) sums
    np.testing.assert_allclose(g_op, op, atol=2e-5)
    np.testing.assert_allclose(g_dep, dep, atol=2e-5)
    np.testing.assert_allclose(g_rgb, rgb, atol=2e-5)
    np.testing.assert_allclose(g_ws, ws, atol=2e-6)
    # early-termination point may move by one sample when T crosses 1e-4 within rounding
    assert np.abs(g_tot.astype(np.int64) - tot).max() <= 1
    assert (g_tot != tot).mean() < 0.02

    go, gd = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    gr, gw = rng.standard_normal((n, 3)).astype(np.float32), rng.standard_normal(S).astype(np.float32)
    dsig, drgbs = oracle.composite_train_bwd(go, gd, gr, gw, sig, rgbs, deltas, ts, rays_a, 1e-4)
    g_dsig, g_drgbs = ops.composite_train_bwd(T(go), T(gd), T(gr), T(gw), T(sig), T(rgbs), T(deltas), T(ts), T(rays_a), 1e-4)
    g_dsig, g_drgbs = N(g_dsig), N(g_drgbs).astype(np.float32)
    same_active = g_tot == tot
    ray_of = np.empty(S, np.int64)
    for r, s0, c in rays_a:
        ray_of[s0:s0 + c] = r
    m = same_active[ray_of]
    scale = np.abs(dsig).max()
    assert np.abs(g_dsig[m] - dsig[m]).max() <= 1e-3 * scale
    tol = 2e-3 if half else 1e-5
    assert np.abs(g_drgbs[m] - drgbs[m].astype(np.float32)).max() <= tol * max(1.0, np.abs(drgbs).max())


def test_volume_renderer_autograd(oracle):
    from modules.volume_train import VolumeRenderer
    rng = np.random.default_rng(31)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, 300, 120, False, True)
    vr = VolumeRenderer()
    s, c = T(sig).requires_grad_(True), T(rgbs).requires_grad_(True)
    total, opacity, depth, rgb, ws = vr(s, c, T(deltas), T(ts), T(rays_a), 1e-4)
    tgt = torch.rand_like(rgb)
    loss = ((rgb + (1 - opacity)[:, None] - tgt) ** 2).mean()
    loss.backward()
    n = rays_a.shape[0]
    g_rgb = N(2 * (rgb + (1 - opacity)[:, None] - tgt) / (3 * n))
    g_op = -g_rgb.sum(1)
    dsig, drgbs = oracle.composite_train_bwd(g_op, np.zeros(n, np.float32), g_rgb, np.zeros_like(sig), sig, rgbs,
                                             deltas, ts, rays_a, 1e-4)
    assert np.abs(N(s.grad) - dsig).max() <= 1e-3 * np.abs(dsig).max()
    assert int(total) == int(oracle.composite_train_fwd(sig, rgbs, deltas, ts, rays_a, 1e-4)[0].sum())


# ---- a9 -------------------------------------------------------------------------------------------
def test_composite_test(ops, oracle):
    rng = np.random.default_rng(32)
    n_rays, A = 500, 300
    alive = rng.permutation(n_rays)[:A].astype(np.int64)
    steps = rng.integers(0, 9, A)
    pack = np.stack([np.cumsum(steps) - steps, steps], 1).astype(np.int64)
    S = int(steps.sum())
    sig = (rng.random(S) * 2000).astype(np.float32)
    rgbs = rng.random((S, 3)).astype(np.float16)
    deltas = np.full(S, 1.7320508075688772 / 1024, np.float32)
    ts = rng.random(S).astype(np.float32)
    op0 = (rng.random(n_rays) * 0.5).astype(np.float32)
    r_alive, r_op, r_dep, r_rgb = alive.copy(), op0.copy(), np.zeros(n_rays, np.float32), np.zeros((n_rays, 3), np.float32)
    oracle.composite_test(sig, rgbs, deltas, ts, pack, r_alive, 1e-4, r_op, r_dep, r_rgb)
    g_alive, g_op, g_dep, g_rgb = T(alive), T(op0), torch.zeros(n_rays, device=DEV), torch.zeros(n_rays, 3, device=DEV)
    ops.composite_test(T(sig), T(rgbs), T(deltas), T(ts), T(pack), g_alive, 1e-4, g_op, g_dep, g_rgb)
    assert np.array_equal(N(g_alive), r_alive)
    np.testing.assert_allclose(N(g_op), r_op, atol=1e-6)
    np.testing.assert_allclose(N(g_dep), r_dep, atol=1e-6)
    np.testing.assert_allclose(N(g_rgb), r_rgb, atol=1e-6)


# ---- grid helpers / optimizer -------------------------------------------------------------------------
def test_packbits_morton_bit_exact(ops, oracle):
    rng = np.random.default_rng(33)
    grid = rng.standard_normal(128 ** 3).astype(np.float32)
    bits = torch.zeros(128 ** 3 // 8, device=DEV, dtype=torch.uint8)
    ops.packbits(T(grid), 0.25, bits)
    assert np.array_equal(N(bits), oracle.packbits(grid, 0.25))
    coords = rng.integers(0, 128, (100003, 3)).astype(np.int32)
    idx = ops.morton3d(T(coords))
    assert np.array_equal(N(idx), oracle.morton3d(coords))
    assert np.array_equal(N(ops.morton3d_invert(idx)), coords)


@pytest.mark.parametrize("n", [1000, 11420064 // 8 + 3])
def test_adam_fused(ops, oracle, n):
    rng = np.random.default_rng(34)
    p = rng.standard_normal(n).astype(np.float32)
    m, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
    gp, gm, gv = T(p), T(m), T(v)
    shadow = torch.zeros(n, device=DEV, dtype=torch.float16)
    found = torch.zeros(1, device=DEV, dtype=torch.int32)
    for step in range(1, 4):
        g = (rng.standard_normal(n) * 65536).astype(np.float32)
        gg = T(g)
        ops.check_finite(gg, found)
        ops.adam_step(gp, gg, gm, gv, 1e-2, step, inv_scale=1 / 65536, param_f16=shadow, found_inf=found, zero_grad=True)
        oracle.adam_step(p, g, m, v, 1e-2, step, inv_scale=1 / 65536)
        assert not N(gg).any()
    # same fp32 formula; sqrt/div rounding may differ in the last ulp and nvcc contracts into fma
    np.testing.assert_allclose(N(gp), p, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(N(gv), v, rtol=2e-6)
    assert np.array_equal(N(shadow), N(gp).astype(np.float16))
    # inf -> step skipped
    before = N(gp).copy()
    g = T(np.full(n, np.nan, np.float32))
    ops.check_finite(g, found)
    assert int(found) == 1
    ops.adam_step(gp, g, gm, gv, 1e-2, 4, found_inf=found)
    assert np.array_equal(N(gp), before)


@pytest.mark.parametrize("saved", [False, True])
@pytest.mark.parametrize("emb_half", [True, False])
@pytest.mark.parametrize("n", [1, 128, 5000, 40000])
def test_mlp_bwd_tcgen05_matches_oracle(ops, oracle, emb_half, n, saved):
    _mlp_bwd_matches_oracle(ops, oracle, emb_half, n, saved, "xavier")


@pytest.mark.parametrize("saved", [False, True])
@pytest.mark.parametrize("emb_half", [True, False])
@pytest.mark.parametrize("n", [1, 128, 5000, 40000])
def test_mlp_bwd_tcgen05_matches_oracle_trained(ops, oracle, emb_half, n, saved):
    """The same comparison on the finite regimes of tests/mlp_tolerance.py::trained_inputs; on its probe rows the
    TruncExp gradient (r16(dsig exp(+-15)) where h0 is clamped) must also reach dL/demb exactly, through the
    recompute and the saved-activation backward."""
    _mlp_bwd_matches_oracle(ops, oracle, emb_half, n, saved, "trained")


def _mlp_bwd_matches_oracle(ops, oracle, emb_half, n, saved, magnitude):
    rng = np.random.default_rng(35)
    emb = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16 if emb_half else np.float32)
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    ws = _weights(rng)
    dsig = (rng.standard_normal(n) * 0.1).astype(np.float32)
    drgb = (rng.standard_normal((n, 3)) * 0.1).astype(np.float16)
    rows = None
    if magnitude == "trained":
        from mlp_tolerance import trained_inputs
        emb, dirs, ws, dsig, drgb, rows = trained_inputs(n, 35, np.float16 if emb_half else np.float32)
    demb_ref, gw_ref = oracle.mlp_bwd(emb, dirs, ws, dsig, drgb)
    save = None
    if saved:   # backward restarting from the activations the forward kept (h + fp16 rgb) instead of recomputing
        sig_f, rgb_f, save = ops.mlp_fwd(T(emb), T(dirs), [T(w) for w in ws], with_save=True)
        sig_n, rgb_n = ops.mlp_fwd(T(emb), T(dirs), [T(w) for w in ws])
        assert torch.equal(sig_f, sig_n) and torch.equal(rgb_f, rgb_n)       # saving does not change the outputs
        kept = save.view(torch.float16)
        assert torch.equal(kept[n * 16:n * 16 + n * 4].view(n, 4)[:, :3], rgb_f)
    demb, gw = ops.mlp_bwd(T(emb), T(dirs), [T(w) for w in ws], T(dsig), T(drgb), save=save)
    demb, gw = N(demb).astype(np.float32), N(gw)
    if rows is not None:
        from test_gpu_mlp_magnitudes import check_probe_rows
        sig_k, _ = ops.mlp_fwd(T(emb), T(dirs), [T(w) for w in ws])
        assert check_probe_rows(demb, N(sig_k), dsig, rows) > 0
    demb_ref = demb_ref.astype(np.float32)
    # Error model (scripts/measure_mlp_bwd_error.py).  Every intermediate gradient is rounded to fp16 on both
    # sides and the tensor core sums K in a different order, so individual roundings flip by one fp16 ulp: the bulk of
    # the elements agrees to ~2e-5 of the tensor's max (asserted on the 99.9th percentile at 1e-4 = 5x measured).  The
    # few large deviations are not rounding noise but ReLU-mask flips: a hidden pre-activation within an ulp of zero is
    # positive on one side and zero on the other, which switches a whole path of the backward on or off; measured
    # up to 3.0e-3 of max on demb and on the dW3 / dW4 blocks at n = 40000, asserted at 5e-3.
    err = np.abs(demb - demb_ref)
    assert np.percentile(err, 99.9) <= 1e-4 * np.abs(demb_ref).max()
    assert err.max() <= 5e-3 * np.abs(demb_ref).max()
    assert np.abs(gw - gw_ref).max() <= 5e-3 * np.abs(gw_ref).max()
    big = np.abs(gw_ref) > 0.05 * np.abs(gw_ref).max()
    assert np.median(np.abs(gw[big] - gw_ref[big]) / np.abs(gw_ref[big])) < 1e-4       # measured ~2e-5
    # per-layer blocks must all be populated (catches a transposed / misplaced dW block)
    offs = np.cumsum([0, 2048, 1024, 2048, 4096, 192])
    for a, b in zip(offs[:-1], offs[1:]):
        blk, ref = gw[a:b], gw_ref[a:b]
        assert np.abs(blk - ref).max() <= 5e-3 * max(np.abs(ref).max(), 1e-6), (a, b)


def test_distortion_loss(ops, oracle):
    rng = np.random.default_rng(36)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, 600, 200, False, False)
    S = sig.shape[0]
    ws = (rng.random(S) * 0.05).astype(np.float32)
    ref = oracle.distortion_fwd(ws, deltas, ts, rays_a)
    got = N(ops.distortion_fwd(T(ws), T(deltas), T(ts), T(rays_a)))
    # 2*(wts_inc*ws_exc - ws_inc*wts_exc) subtracts nearly equal fp32 products (the reference's formula,
    # distortion.py:64), so fp32 results carry ~1e-3 relative noise whatever the summation order; both the
    # oracle and the kernel are compared with an fp64 evaluation of the same formula
    w64, t64 = ws.astype(np.float64), ts.astype(np.float64)
    ref64 = np.zeros(rays_a.shape[0])
    for ray, s0, c in rays_a:
        w, t, d = w64[s0:s0 + c], t64[s0:s0 + c], deltas[s0:s0 + c].astype(np.float64)
        wi, wti = np.cumsum(w), np.cumsum(w * t)
        ref64[ray] = (2 * (wti * (wi - w) - wi * (wti - w * t)) + w * w * d / 3).sum()
    np.testing.assert_allclose(got, ref64, rtol=5e-3, atol=1e-6)
    np.testing.assert_allclose(ref, ref64, rtol=5e-3, atol=1e-6)
    g = rng.standard_normal(rays_a.shape[0]).astype(np.float32)
    dref = oracle.distortion_bwd(g, ws, deltas, ts, rays_a)
    dgot = N(ops.distortion_bwd(T(g), T(ws), T(deltas), T(ts), T(rays_a)))
    assert np.abs(dgot - dref).max() <= 1e-3 * np.abs(dref).max()
    from modules.distortion import distortion_loss
    w = T(ws).requires_grad_(True)
    distortion_loss({'ws': w, 'deltas': T(deltas), 'ts': T(ts), 'rays_a': T(rays_a)}).mean().backward()
    assert np.abs(N(w.grad) - oracle.distortion_bwd(np.full(rays_a.shape[0], 1 / rays_a.shape[0], np.float32),
                                                    ws, deltas, ts, rays_a)).max() <= 1e-3 * np.abs(N(w.grad)).max()


def test_packbits_device_threshold(ops, oracle):
    rng = np.random.default_rng(37)
    grid = rng.standard_normal(128 ** 3).astype(np.float32)
    for mean, thr in ((0.3, 5.9), (7.0, 5.9), (float('nan'), 5.9)):
        bits = torch.full((128 ** 3 // 8,), 255, device=DEV, dtype=torch.uint8)
        ops.packbits(T(grid), thr, bits, mean_dev=torch.tensor([mean], device=DEV))
        eff = min(mean, thr)  # python semantics of networks.py:288-290 (NaN mean -> NaN threshold -> no bits)
        want = oracle.packbits(grid, eff) if eff == eff else np.zeros(128 ** 3 // 8, np.uint8)
        assert np.array_equal(N(bits), want)


@pytest.mark.parametrize("half", [False, True])
def test_hash_generic_feature_width(ops, oracle, half):
    """--deployment configuration of the reference (train.py:88-99): L=4, F=4, 32->128, T=2^21, all dense."""
    rng = np.random.default_rng(38)
    lay = make_hash_layout(2 ** 21, 4, 32, 128, 4)
    n = 3000
    xyz = rng.random((n, 3), dtype=np.float32)
    table = rng.standard_normal(lay.total_param_size).astype(np.float16 if half else np.float32)
    ref = oracle.hash_encode_fwd(xyz, table, lay)
    got = N(ops.hash_encode_fwd(T(xyz), T(table), lay.as_ctypes(), lay.out_dim))
    assert np.array_equal(got.view(np.uint8), ref.view(np.uint8))
    dout = rng.standard_normal((n, lay.out_dim)).astype(table.dtype)
    gref = oracle.hash_encode_bwd(xyz, dout, lay)
    g = torch.zeros(lay.total_param_size, device=DEV)
    ops.hash_encode_bwd(T(xyz), T(dout), lay.as_ctypes(), g)
    np.testing.assert_allclose(N(g), gref, rtol=1e-3, atol=1e-4)


def test_deployment_model_config_trains():
    """NGP(**deployment config) falls back to nn.Linear MLPs + generic-F hash kernels and can take a step."""
    from modules.networks import NGP
    from taichi_nerfs_b200.trainer import NGPTrainer
    from oracle.train_step import make_rays
    m = NGP(scale=0.5, levels=4, feature_per_level=4, base_res=32, max_res=128, log2_T=21, xyz_net_width=16,
            rgb_net_width=16, rgb_net_depth=1).cuda()
    assert not m._fusable(next(m.parameters()))
    with torch.no_grad():
        m.density_bitfield.fill_(255)
    o, d = make_rays(512, seed=13)
    tr = NGPTrainer(m)
    before = m.pos_encoder.hash_table.detach().clone()
    loss, res = tr.step(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), torch.rand(512, 3, device='cuda'))
    assert torch.isfinite(loss) and (m.pos_encoder.hash_table != before).any()


def test_march_frame_single_pass(ops, oracle, rays_factory, lego_bitfield):
    """Single-pass test-time march == oracle training march with zero noise, per ray (row order is arbitrary)."""
    _check_frame_march(ops, oracle, rays_factory, lego_bitfield, MARCH_CFGS[0])


@pytest.mark.parametrize("cfg", MARCH_CFGS[1:], ids=MARCH_IDS[1:])
def test_march_frame_single_pass_configs(ops, oracle, rays_factory, lego_bitfield, cfg):
    """The same at the other march configurations (cascades, exp_step_factor, occupancy)."""
    _check_frame_march(ops, oracle, rays_factory, lego_bitfield, cfg)


def _check_frame_march(ops, oracle, rays_factory, lego_bitfield, cfg):
    n = 5003
    o, d, bits = _march_inputs(cfg, n, 40, np.random.default_rng(40), rays_factory, lego_bitfield)
    sc, casc, esf = cfg["scale"], cfg["cascades"], cfg["esf"]
    hits = oracle.ray_aabb_intersect(o, d, sc)
    ra, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, np.zeros(n, np.float32), casc, sc,
                                                            esf, 128, 1024)
    assert S > 0
    cap = S + 100
    counter = torch.zeros(2, device=DEV, dtype=torch.int32)
    g_ra = torch.zeros(n, 3, device=DEV, dtype=torch.int32)
    bufs = [torch.zeros(cap, 3, device=DEV), torch.zeros(cap, 3, device=DEV), torch.zeros(cap, device=DEV), torch.zeros(cap, device=DEV)]
    ops.raymarching_frame(T(o), T(d), T(hits), T(bits), casc, sc, esf, 128, 1024, counter, g_ra, *bufs)
    assert N(counter).tolist() == [S, 0]
    g_ra = N(g_ra)
    assert np.array_equal(g_ra[:, 0], ra[:, 0]) and np.array_equal(g_ra[:, 2], ra[:, 2])
    g_x, g_d, g_dl, g_t = [N(b) for b in bufs]
    # gather the GPU rows back into ray order and compare bit-exactly
    order = np.concatenate([np.arange(s0, s0 + c) for _, s0, c in g_ra if c > 0])
    assert np.array_equal(np.sort(order), np.arange(S))  # the reserved ranges tile [0, S) exactly
    for a, b in ((g_x, xyzs), (g_d, dirs), (g_dl, deltas), (g_t, ts)):
        assert np.array_equal(a[order].view(np.uint32), b.view(np.uint32))
    # capacity overflow: rays are dropped and counted, never written out of bounds
    counter.zero_()
    small = [torch.zeros(S // 3, 3, device=DEV), torch.zeros(S // 3, 3, device=DEV), torch.zeros(S // 3, device=DEV), torch.zeros(S // 3, device=DEV)]
    ops.raymarching_frame(T(o), T(d), T(hits), T(bits), casc, sc, esf, 128, 1024, counter, T(ra * 0), *small)
    assert N(counter)[1] > 0


@pytest.mark.parametrize("dense", [False, True])
def test_ray_head_fused_equals_separate_kernels(ops, oracle, dense):
    """composite fwd + bg + MSE + composite bwd in one launch == the three separate kernels == the oracle."""
    import ctypes as C
    from taichi_nerfs_b200 import _lib
    rng = np.random.default_rng(41)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, 500, 200, dense, True)
    rays_a[:, 0] = np.arange(500)
    n, S = rays_a.shape[0], sig.shape[0]
    gt = rng.random((n, 3)).astype(np.float32)
    scale = 1024.0
    tot, op, dep, rgb, ws = oracle.composite_train_fwd(sig, rgbs, deltas, ts, rays_a, 1e-4)
    out = rgb + (1 - op)[:, None]
    diff = out - gt
    g_rgb = (scale * 2 * diff / (3 * n)).astype(np.float32)
    g_op = -g_rgb.sum(1)
    dsig_ref, drgbs_ref = oracle.composite_train_bwd(g_op, np.zeros(n, np.float32), g_rgb, np.zeros(S, np.float32),
                                                     sig, rgbs, deltas, ts, rays_a, 1e-4)
    t_sig, t_rgbs, t_dl, t_ra, t_gt = T(sig), T(rgbs), T(deltas), T(rays_a), T(gt)
    loss_sum = torch.zeros(1, device=DEV)
    o_op, o_rgb = torch.zeros(n, device=DEV), torch.zeros(n, 3, device=DEV)
    dsig, drgbs = torch.zeros(S, device=DEV), torch.zeros(S, 3, device=DEV, dtype=torch.float16)
    p = lambda t: C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.load().ngp_ray_head_fused(p(t_sig), p(t_rgbs), 1, p(t_dl), p(t_ra), p(t_gt), 1.0, scale, None, 1e-4,
                                              p(loss_sum), p(o_op), p(o_rgb), p(dsig), p(drgbs), n, st))
    np.testing.assert_allclose(N(o_op), op, atol=2e-5)
    np.testing.assert_allclose(N(o_rgb), out, atol=3e-5)
    assert abs(float(loss_sum) - float((diff.astype(np.float64) ** 2).sum())) < 1e-3 * float((diff ** 2).sum())
    assert np.abs(N(dsig) - dsig_ref).max() <= 2e-3 * np.abs(dsig_ref).max()
    assert np.abs(N(drgbs).astype(np.float32) - drgbs_ref.astype(np.float32)).max() <= 3e-3 * max(1.0, np.abs(drgbs_ref.astype(np.float32)).max())


@pytest.mark.gpu
def test_sample_ray_batch_bit_exact(ops, oracle):
    """ngp_sample_ray_batch == oracle for both index sources (given indices / Philox by (seed, step, ray))."""
    rng = np.random.default_rng(9)
    n_img, n_pix, n = 13, 40 * 30, 10007
    poses = rng.standard_normal((n_img, 3, 4)).astype(np.float32)
    dirs = rng.standard_normal((n_pix, 3)).astype(np.float32)
    bank = rng.random((n_img, n_pix, 3)).astype(np.float32)
    tb, tp, td = (torch.from_numpy(a).cuda() for a in (bank, poses, dirs))
    step_dev = torch.tensor([77], device="cuda", dtype=torch.int32)
    for kw_gpu, kw_cpu in [
        (dict(seed=2**40 + 5, step=9), dict(seed=2**40 + 5, step=9)),
        (dict(seed=3, step_dev=step_dev), dict(seed=3, step=77)),
        (dict(seed=3, fixed_img=4), dict(seed=3, fixed_img=4)),
    ]:
        got = ops.sample_ray_batch(tb, tp, td, n, return_indices=True, **kw_gpu)
        want = oracle.sample_ray_batch(bank, poses, dirs, n, **kw_cpu)
        for k in ("img_idxs", "pix_idxs", "rays_o", "rays_d", "rgb", "noise"):
            np.testing.assert_array_equal(got[k].cpu().numpy(), want[k], err_msg=k)
    ii = torch.from_numpy(rng.integers(0, n_img, n)).cuda()
    pi = torch.from_numpy(rng.integers(0, n_pix, n)).cuda()
    got = ops.sample_ray_batch(tb, tp, td, n, img_idxs=ii, pix_idxs=pi, with_noise=False)
    want = oracle.sample_ray_batch(bank, poses, dirs, n, img_idxs=ii.cpu().numpy(), pix_idxs=pi.cpu().numpy())
    for k in ("rays_o", "rays_d", "rgb"):
        np.testing.assert_array_equal(got[k].cpu().numpy(), want[k], err_msg=k)
    assert got["noise"] is None
    assert ops.sample_ray_batch(tb, tp, td, 0)["rays_o"].shape == (0, 3)


# ---- fast_hash / under_hash known-answer test on the CUDA kernels ---------------------------------------------
@pytest.mark.parametrize("max_res", [1024, 4096])
def test_hash_index_known_answers_cuda(ops, max_res):
    """CUDA hash forward (fp32 table) against hash_encoder.py:43-71,108-139 evaluated with Python integers
    (tests/hash_kat.py): the table stores its own entry index, so the output reveals every index touched."""
    import hash_kat as K
    from taichi_nerfs_b200.layout import make_hash_layout
    lay = make_hash_layout(2 ** 19, 16, 16, max_res, 2)
    want = K.expected(lay, K.POINTS)
    pts = np.tile(K.POINTS, (80, 1))                      # > one 512-sample CTA tile, repeated cells exercise the run reuse
    got = N(ops.hash_encode_fwd(T(pts), T(K.index_table(lay).reshape(-1)), lay.as_ctypes(), 32)).astype(np.float64)
    np.testing.assert_allclose(got, np.tile(want, (80, 1)), rtol=2e-6, atol=0.5)


# ---- f1: fused occupancy-grid update ---------------------------------------------------------------------------
@pytest.mark.parametrize("warmup", [True, False])
@pytest.mark.parametrize("cascades,scale", [(1, 0.5), (3, 2.0), (5, 8.0), (3, 1.5)])
def test_fused_grid_update_matches_oracle(ops, oracle, warmup, cascades, scale):
    """Cell pick + jittered positions (networks.py:168-209, 263-271): bit-exact vs the oracle restatement (same Philox
    draws); scatter-max + EMA-max + mean + packbits (:272-290): grid bit-exact, mean within 1 fp32 ulp, bitfield equal."""
    G = 128
    rng = np.random.default_rng(17 + cascades)
    grid = (rng.random((cascades, G ** 3)) ** 6 * 40).astype(np.float32)        # ~10 % above the 5.91 threshold
    grid[:, rng.integers(0, G ** 3, 20000)] = -1.0                               # cells no camera sees
    thr, M, seed, step = 0.01 * 1024 / 3 ** 0.5, G ** 3 // 4, 0x6E6770, 7
    ws = ops.grid_workspace(cascades, G, "cuda")
    g_dev = T(grid)
    idx, xyz = ops.grid_sample_cells(g_dev, scale, thr, warmup, M, seed, step, ws)
    idx_ref, xyz_ref = oracle.grid_sample_cells(grid, scale, thr, warmup, M, seed, step)
    np.testing.assert_array_equal(N(idx), idx_ref)
    np.testing.assert_array_equal(N(xyz), xyz_ref)
    if not warmup:   # the occupied half really is occupied, the uniform half covers the grid
        per = 2 * M
        for c in range(cascades):
            occ = idx_ref[c * per + M:(c + 1) * per]
            assert (grid[c, occ] > thr).all()
    dens = (rng.random(idx_ref.size) ** 4 * 30).astype(np.float32)
    mean = torch.zeros(1, device="cuda")
    bits = torch.zeros(cascades * G ** 3 // 8, device="cuda", dtype=torch.uint8)
    ops.grid_update(g_dev, idx, T(dens), thr, 0.95, ws, mean, bits)
    new_ref, mean_ref, bits_ref = oracle.grid_update(grid, idx_ref, dens, thr)
    np.testing.assert_array_equal(N(g_dev), new_ref)
    assert abs(float(mean) - float(mean_ref)) <= 1.2e-7 * abs(float(mean_ref))
    np.testing.assert_array_equal(N(bits), bits_ref)


def test_fused_grid_update_no_occupied_cells_and_erode(ops, oracle):
    """No cell above the threshold -> the occupied half is empty (index -1, networks.py:193) and ignored; erode uses the
    per-cell decay clamp(decay^(1/count), 0.1, 0.95) (:274-275)."""
    G = 128
    rng = np.random.default_rng(5)
    grid = (rng.random((1, G ** 3)) * 0.5).astype(np.float32)
    thr, M = 5.9, G ** 3 // 4
    ws = ops.grid_workspace(1, G, "cuda")
    g_dev = T(grid)
    idx, xyz = ops.grid_sample_cells(g_dev, 0.5, thr, False, M, 1, 0, ws)
    idx_ref, xyz_ref = oracle.grid_sample_cells(grid, 0.5, thr, False, M, 1, 0)
    assert (idx_ref[M:] == -1).all()
    np.testing.assert_array_equal(N(idx), idx_ref)
    np.testing.assert_array_equal(N(xyz), xyz_ref)
    count = (rng.random((1, G ** 3)) * 0.9 + 0.05).astype(np.float32)
    dens = rng.random(idx_ref.size).astype(np.float32)
    mean = torch.zeros(1, device="cuda")
    bits = torch.zeros(G ** 3 // 8, device="cuda", dtype=torch.uint8)
    ops.grid_update(g_dev, idx, T(dens), thr, 0.95, ws, mean, bits, count_grid=T(count))
    new_ref, mean_ref, bits_ref = oracle.grid_update(grid, idx_ref, dens, thr, count_grid=count)
    np.testing.assert_allclose(N(g_dev), new_ref, rtol=2e-6)   # powf: 1-2 ulp between libm and CUDA
    np.testing.assert_array_equal(N(bits), bits_ref)


# ---- compacting renderer: round march (resume points, per-ray cap over the frame) ----------------------------------
# garden scale, every cell occupied, rays from inside the box: every ray has more than max_samples candidate positions
GARDEN_FULL = dict(scale=16.0, cascades=6, esf=1 / 256, occ="full")


@pytest.mark.parametrize("cfg", MARCH_CFGS + [GARDEN_FULL], ids=MARCH_IDS + ["6casc_full_capped"])
def test_round_march_equals_full_march(ops, oracle, lego_bitfield, rays_factory, cfg):
    """The per-round march of the compacting frame renderer (persistent warps over a live list, <= limit samples per
    ray and round, resume at t_cur, a per-ray count that caps a ray at max_samples over all rounds) must emit, ray by
    ray, exactly the samples of the oracle's one-shot march with zero noise (bit-exact t, delta, xyz and count),
    whatever the rounds, at every march configuration."""
    import ctypes as C
    from taichi_nerfs_b200 import _lib
    L = _lib.load()
    n = 6000
    o_np, d_np, bits_np = _march_inputs(cfg, n, 77, np.random.default_rng(77), rays_factory, lego_bitfield)
    sc, casc, esf = cfg["scale"], cfg["cascades"], cfg["esf"]
    hits_np = oracle.ray_aabb_intersect(o_np, d_np, sc)
    ra, xyz_ref, dirs_ref, dl_ref, ts_ref, S = oracle.raymarching_train(o_np, d_np, hits_np, bits_np,
                                                                       np.zeros(n, np.float32), casc, sc, esf, 128, 1024)
    o, d, bits, hits = T(o_np), T(d_np), T(bits_np), T(hits_np)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    cap = 64 * n
    t_cur = torch.where(hits[:, 0] > 0, hits[:, 0], torch.full_like(hits[:, 0], -1.0)).contiguous()
    n_marched = torch.zeros(n, device="cuda", dtype=torch.int32)
    alive = torch.arange(n, device="cuda", dtype=torch.int32)
    state = torch.zeros(8, device="cuda", dtype=torch.int32)
    r_a = torch.zeros(n, 3, device="cuda", dtype=torch.int32)
    xyz, dirs = torch.empty(cap, 3, device="cuda"), torch.empty(cap, 3, device="cuda")
    dl, ts = torch.empty(cap, device="cuda"), torch.empty(cap, device="cuda")
    rows_ray, rows_t, rows_dl, rows_xyz = [], [], [], []
    schedule = [4, 8, 16, 3, 64, 128, 256, 512]
    rounds = 0
    while not bool(((t_cur == float("inf")) | (t_cur < 0)).all()) and rounds < 64:
        limit = schedule[rounds] if rounds < len(schedule) else 512
        rounds += 1
        state.zero_()
        state[2] = n                                                  # every ray stays on the live list
        _lib.check(L.ngp_raymarching_round(p(o), p(d), p(hits), p(bits), casc, 128, sc, esf, limit, 1024, p(alive),
                                           p(state), p(t_cur), p(n_marched), p(r_a), p(xyz), p(dirs), p(dl), p(ts),
                                           n, cap, st))
        rows = int(state[0])
        eff = max(1, min(limit, cap // n))
        r_np = N(r_a)
        assert (r_np[:, 2] <= eff).all() and int(r_np[:, 2].sum()) == rows
        ray_of, idx = _row_order(r_np)
        assert np.array_equal(np.sort(idx), np.arange(rows))          # the reserved ranges tile [0, rows)
        rows_ray.append(ray_of)
        rows_t.append(N(ts)[idx])
        rows_dl.append(N(dl)[idx])
        rows_xyz.append(N(xyz)[idx])
    done = (t_cur == float("inf")) | (t_cur < 0)
    assert bool(done.all()), "every ray must have left the box or reached max_samples"
    np.testing.assert_array_equal(N(n_marched), ra[:, 2])              # per-ray sample count == the capped march's
    # rows of all rounds, stably grouped by ray (rounds in order) == the oracle's rows, which are in ray order
    order = np.argsort(np.concatenate(rows_ray), kind="stable")
    for got, want in ((rows_t, ts_ref), (rows_dl, dl_ref), (rows_xyz, xyz_ref)):
        got = np.concatenate(got)[order]
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert S > 30000
    if cfg["occ"] == "full":
        assert (ra[:, 2] == 1024).mean() > 0.9            # the per-ray cap is what ends these rays
