"""CPU-only validation of the oracle itself (the reference ships no tests or golden vectors, so the
oracle is cross-checked against independent numpy / torch restatements, fp64 finite differences and
algebraic properties)."""
import numpy as np
import pytest
import torch

from taichi_nerfs_b200.layout import make_hash_layout


# ------------------------------------------------------------------------------------------------
# independent numpy restatement of the hash encoder (vectorised over samples, one level at a time)
def np_hash_encode(xyz, table, lay, half):
    n = xyz.shape[0]
    F = lay.feat_dim
    tab = table.reshape(-1, F)
    out = np.zeros((n, lay.levels, F), np.float16 if half else np.float32)
    for l in range(lay.levels):
        scale = np.float32(lay.scales[l])
        res = np.uint32(lay.resolutions[l])
        pos = (xyz * scale).astype(np.float32) + np.float32(0.5)
        g = np.floor(pos).astype(np.int64).astype(np.uint32)
        gf = g.astype(np.float16).astype(np.float32) if half else g.astype(np.float32)
        frac = pos - gf
        acc = np.zeros((n, F), np.float16 if half else np.float32)
        for c in range(8):
            w = np.ones(n, np.float32)
            p = []
            for d in range(3):
                if c & (1 << d):
                    p.append(g[:, d] + np.uint32(1))
                    w = w * frac[:, d]
                else:
                    p.append(g[:, d])
                    w = w * (np.float32(1) - frac[:, d])
            if l < lay.begin_fast_hash_level:
                h = p[0] + p[1] * res + p[2] * (res * res)
            else:
                h = p[0] ^ (p[1] * np.uint32(2654435761)) ^ (p[2] * np.uint32(805459861))
            idx = lay.offsets[l] + (h % np.uint32(lay.map_sizes[l])).astype(np.int64)
            prod = w[:, None] * tab[idx].astype(np.float32)
            if half:
                acc = (acc.astype(np.float64) + prod.astype(np.float16).astype(np.float64)).astype(np.float16)
            else:
                acc = acc + prod
        out[:, l] = acc
    return out.reshape(n, -1)


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("max_res", [1024, 4096])
def test_hash_fwd_matches_numpy(oracle, half, max_res):
    rng = np.random.default_rng(1)
    lay = make_hash_layout(2 ** 19, 16, 16, max_res, 2)
    n = 2000
    xyz = rng.random((n, 3), dtype=np.float32)
    xyz[:8] = np.array([[0, 0, 0], [1, 1, 1], [0, 1, 0.5], [1, 0, 0], [0.5, 0.5, 0.5], [1, 1, 0], [0, 0, 1],
                        [0.999999, 1e-7, 0.25]], np.float32)
    if half:
        table = ((rng.random(lay.total_param_size, dtype=np.float32) * 2 - 1) * 1e-4).astype(np.float16)
    else:
        table = rng.random(lay.total_param_size, dtype=np.float32)
    with np.errstate(over="ignore"):
        ref = np_hash_encode(xyz, table, lay, half)
    got = oracle.hash_encode_fwd(xyz, table, lay)
    assert got.dtype == ref.dtype
    if half:
        assert np.array_equal(got.view(np.uint16), ref.view(np.uint16))
    else:
        np.testing.assert_allclose(got, ref, rtol=2e-6, atol=1e-7)  # summation order of 8 terms


@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_is_adjoint_of_fwd(oracle, half):
    """<encode(table), dout> == <table, bwd(dout)> (the encoder is linear in the table)."""
    rng = np.random.default_rng(2)
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
    n = 3000
    xyz = rng.random((n, 3), dtype=np.float32)
    table = rng.standard_normal(lay.total_param_size).astype(np.float32)
    dout = rng.standard_normal((n, 32)).astype(np.float32)
    if half:
        dout = dout.astype(np.float16)
    out = oracle.hash_encode_fwd(xyz, table, lay).astype(np.float64)  # fp32 forward = exact linear map
    grad = oracle.hash_encode_bwd(xyz, dout, lay)
    lhs = float((out * dout.astype(np.float64)).sum())
    rhs = float((table.astype(np.float64) * grad.astype(np.float64)).sum())
    assert abs(lhs - rhs) <= 2e-4 * max(abs(lhs), 1.0)


def test_hash_bwd_input_matches_finite_difference(oracle):
    rng = np.random.default_rng(3)
    lay = make_hash_layout(2 ** 14, 4, 4, 32, 2)  # coarse grid: FD stays inside one cell
    n = 64
    xyz = (rng.random((n, 3)) * 0.9 + 0.05).astype(np.float32)
    table = rng.standard_normal(lay.total_param_size).astype(np.float32)
    dout = rng.standard_normal((n, lay.out_dim)).astype(np.float32)
    dx = oracle.hash_encode_bwd_input(xyz, table, dout, lay)
    eps = 1e-3
    for d in range(3):
        xp, xm = xyz.copy(), xyz.copy()
        xp[:, d] += eps
        xm[:, d] -= eps
        fd = ((oracle.hash_encode_fwd(xp, table, lay).astype(np.float64) -
               oracle.hash_encode_fwd(xm, table, lay).astype(np.float64)) * dout).sum(1) / (xp[:, d] - xm[:, d])
        ok = np.isclose(dx[:, d], fd, rtol=5e-2, atol=5e-2)
        assert ok.mean() > 0.8  # samples whose +-eps straddles a cell boundary are excluded


# ------------------------------------------------------------------------------------------------
def test_aabb_matches_numpy(oracle, rays_factory):
    o, d = rays_factory(4096, seed=4)
    d[:10] *= -1  # rays pointing away
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    inv = (1.0 / d).astype(np.float32)
    tmin = ((-0.5 - o) * inv).astype(np.float32)
    tmax = ((0.5 - o) * inv).astype(np.float32)
    t1 = np.minimum(tmin, tmax).max(1)
    t2 = np.maximum(tmin, tmax).min(1)
    ref = np.where((t2 > 0)[:, None], np.stack([np.maximum(t1, np.float32(0.01)), t2], 1), -1.0).astype(np.float32)
    assert np.array_equal(hits, ref)


def test_march_train_properties(oracle, lego_bitfield, rays_factory):
    n = 2048
    o, d = rays_factory(n, seed=5)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = np.random.default_rng(5).random(n, dtype=np.float32)
    rays_a, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, lego_bitfield, noise, 1, 0.5, 0.0, 128, 1024)
    assert S == rays_a[:, 2].sum() and xyzs.shape == (S, 3)
    assert np.array_equal(rays_a[:, 0], np.arange(n))
    assert np.array_equal(rays_a[:, 1], np.cumsum(rays_a[:, 2]) - rays_a[:, 2])
    # every sample lies in an occupied cell, inside [t1, t2), on its ray, with the constant Lego step
    ray_of = np.repeat(np.arange(n), rays_a[:, 2])
    assert np.allclose(xyzs, o[ray_of] + ts[:, None] * d[ray_of], atol=1e-6)
    assert np.all(ts < hits[ray_of, 1]) and np.all(ts >= hits[ray_of, 0])
    assert np.all(deltas == np.float32(1.7320508075688772 / 1024))
    cell = np.clip(0.5 * (xyzs / 0.5 + 1) * 128, 0, 127).astype(np.uint32)
    mort = oracle.morton3d(cell.astype(np.int32)).astype(np.int64)
    bits = np.unpackbits(lego_bitfield, bitorder="little")
    assert bits[mort].all()
    # statistics of the trained Lego grid from SURVEY.md §8d (independent numpy march): ~35 % of rays
    # have samples, ~22 samples/ray on average
    assert 0.25 < (rays_a[:, 2] > 0).mean() < 0.45
    assert 15 < S / n < 30
    # ts strictly increasing within a ray
    starts = rays_a[:, 1]
    inc = np.diff(ts) > 0
    boundary = np.zeros(S - 1, bool)
    boundary[starts[1:][(starts[1:] > 0) & (starts[1:] < S)] - 1] = True
    assert np.all(inc | boundary)


def test_march_full_grid_counts(oracle, rays_factory):
    """Fully occupied grid: every step of the chord is a sample => n = number of dt steps in [t1, t2)."""
    n = 256
    o, d = rays_factory(n, seed=6)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    full = np.full(128 ** 3 // 8, 255, np.uint8)
    noise = np.zeros(n, np.float32)
    rays_a, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, full, noise, 1, 0.5, 0.0, 128, 1024)
    dt = np.float32(1.7320508075688772 / 1024)
    for r in range(0, n, 17):
        t, cnt = hits[r, 0], 0
        while 0 <= t < hits[r, 1] and cnt < 1024:
            t = np.float32(t + dt)
            cnt += 1
        assert cnt == rays_a[r, 2]


def test_march_capacity_overflow(oracle, lego_bitfield, rays_factory):
    import ctypes as C
    n = 512
    o, d = rays_factory(n, seed=7)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = np.zeros(n, np.float32)
    rays_a, *_, S = oracle.raymarching_train(o, d, hits, lego_bitfield, noise, 1, 0.5, 0.0, 128, 1024)
    cap = S // 2
    L = oracle.lib()
    counter = np.array([S, n], np.int32)
    ra = rays_a.copy()
    bufs = [np.zeros((cap, 3), np.float32), np.zeros((cap, 3), np.float32), np.zeros(cap, np.float32), np.zeros(cap, np.float32)]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = L.ngp_raymarching_train_write_cpu(p(o), p(d), p(hits), p(lego_bitfield), p(noise), 1, 128, C.c_float(0.5),
                                           C.c_float(0.0), p(counter), p(ra), *[p(b) for b in bufs],
                                           C.c_int64(n), C.c_int64(cap))
    assert rc == 0
    assert counter[0] <= cap and counter[0] == ra[:, 2].sum()
    kept = ra[:, 2] > 0
    assert np.array_equal(ra[kept, 2], rays_a[kept, 2])


def test_march_test_matches_train_samples(oracle, lego_bitfield, rays_factory):
    """Chunked test-time marching visits exactly the samples of a noise-free training march."""
    n = 300
    o, d = rays_factory(n, seed=8)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = np.zeros(n, np.float32)
    rays_a, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, lego_bitfield, noise, 1, 0.5, 0.0, 128, 1024)
    h = hits.copy()
    alive = np.arange(n, dtype=np.int64)
    got = [[] for _ in range(n)]
    for it in range(400):
        if alive.size == 0:
            break
        ri, valid, dl, tt, cnt = oracle.raymarching_test(o, d, h, alive, lego_bitfield, 1, 0.5, 0.0, 128, 4)
        for k, r in enumerate(alive):
            got[r].extend(tt[k * 4:k * 4 + cnt[k]].tolist())
        alive = alive[cnt > 0]
    for r in range(n):
        ref = ts[rays_a[r, 1]:rays_a[r, 1] + rays_a[r, 2]]
        assert np.array_equal(np.asarray(got[r], np.float32), ref), r


# ------------------------------------------------------------------------------------------------
def test_sh_matches_closed_form(oracle):
    rng = np.random.default_rng(9)
    d = rng.standard_normal((100, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    out = oracle.dir_encode(d.astype(np.float32))
    x, y, z = d.T
    assert np.allclose(out[:, 0], 0.28209479177387814)
    assert np.allclose(out[:, 2], 0.48860251190291987 * z, atol=1e-6)
    assert np.allclose(out[:, 6], 0.94617469575755997 * z * z - 0.31539156525251999, atol=1e-6)
    assert np.allclose(out[:, 15], 0.59004358992664352 * x * (-x * x + 3 * y * y), atol=1e-6)
    # real SH of degree l are orthonormal-ish: sum_m Y_lm^2 = (2l+1)/(4 pi) on the unit sphere
    for l, (a, b) in enumerate([(0, 1), (1, 4), (4, 9), (9, 16)]):
        assert np.allclose((out[:, a:b] ** 2).sum(1), (2 * l + 1) / (4 * np.pi), atol=1e-5)


def _torch_mlp_reference(emb, dirs, ws):
    """Independent torch restatement of NGP.forward's network part under autocast semantics
    (fp16 operands, fp32 accumulate, fp16 layer outputs), modules/networks.py:136-166."""
    h16 = lambda t: t.half().float()
    W = [h16(torch.from_numpy(w)) for w in ws]
    e = h16(torch.from_numpy(emb.astype(np.float32)))
    h1 = torch.relu(h16(e @ W[0].T))
    h = h16(h1 @ W[1].T)
    sigma = torch.exp(h[:, 0])
    d = torch.from_numpy(dirs)
    d = d / d.norm(dim=1, keepdim=True)
    d = (d + 1) / 2
    x, y, z = d.unbind(1)
    sh = torch.from_numpy(np.zeros((len(d), 16), np.float32))
    from oracle import oracle as O
    sh = torch.from_numpy(O.dir_encode(d.numpy()))
    x3 = torch.cat([h16(sh), h], 1)
    h3 = torch.relu(h16(x3 @ W[2].T))
    h4 = torch.relu(h16(h3 @ W[3].T))
    o = h16(h4 @ W[4].T)
    rgb = h16(torch.sigmoid(o))
    return sigma.numpy(), rgb.numpy()


def _rand_weights(rng):
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    return [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]


def test_mlp_fwd_matches_torch(oracle):
    rng = np.random.default_rng(10)
    n = 512
    emb = rng.standard_normal((n, 32)).astype(np.float16)
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    ws = _rand_weights(rng)
    sig, rgb = oracle.mlp_fwd(emb, dirs, ws)
    sig_ref, rgb_ref = _torch_mlp_reference(emb, dirs, ws)
    # fp16 rounding of every layer output makes 1-ulp(fp16) flips possible when the fp32 dot
    # product is summed in a different order
    np.testing.assert_allclose(sig, sig_ref, rtol=4e-3)
    np.testing.assert_allclose(rgb.astype(np.float32), rgb_ref, atol=2e-3)


def test_mlp_bwd_matches_torch_autograd(oracle):
    """fp32 autograd through the same fp16-rounded forward values (straight-through on the rounding)."""
    rng = np.random.default_rng(11)
    n = 256
    emb = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    ws = _rand_weights(rng)
    dsig = (rng.standard_normal(n) * 0.1).astype(np.float32)
    drgb = (rng.standard_normal((n, 3)) * 0.1).astype(np.float16)
    demb, gw = oracle.mlp_bwd(emb, dirs, ws, dsig, drgb)

    W = [torch.from_numpy(w).half().float().requires_grad_(True) for w in ws]
    e = torch.from_numpy(emb.astype(np.float32)).requires_grad_(True)
    h1 = torch.relu(e @ W[0].T)
    h = h1 @ W[1].T
    sigma = torch.exp(h[:, 0])
    d = torch.from_numpy(dirs)
    d = (d / d.norm(dim=1, keepdim=True) + 1) / 2
    sh = torch.from_numpy(oracle.dir_encode(d.numpy()))
    h3 = torch.relu(torch.cat([sh, h], 1) @ W[2].T)
    h4 = torch.relu(h3 @ W[3].T)
    rgb = torch.sigmoid(h4 @ W[4].T)
    loss = (sigma * torch.from_numpy(dsig)).sum() + (rgb * torch.from_numpy(drgb.astype(np.float32))).sum()
    loss.backward()
    ref_gw = np.concatenate([w.grad.numpy().reshape(-1) for w in W])
    scale = np.abs(ref_gw).max()
    assert np.abs(gw - ref_gw).max() < 2e-2 * scale
    ref_de = e.grad.numpy()
    assert np.abs(demb.astype(np.float32) - ref_de).max() < 2e-2 * np.abs(ref_de).max()


# ------------------------------------------------------------------------------------------------
def _composite_inputs(rng, n_rays=64, max_n=80, dense=False):
    counts = rng.integers(0, max_n, n_rays)
    counts[0] = 0
    S = int(counts.sum())
    rays_a = np.stack([rng.permutation(n_rays), np.cumsum(counts) - counts, counts], 1).astype(np.int32)
    sig = (rng.random(S) * (40.0 if dense else 3.0)).astype(np.float32)
    rgbs = rng.random((S, 3)).astype(np.float32)
    deltas = np.full(S, 1.7320508075688772 / 1024, np.float32) * (20 if dense else 1)
    ts = np.sort(rng.random(S)).astype(np.float32)
    return rays_a, sig, rgbs, deltas, ts


def _np_composite(rays_a, sig, rgbs, deltas, ts, thr):
    n = rays_a.shape[0]
    op, dep, rgb, ws = np.zeros(n), np.zeros(n), np.zeros((n, 3)), np.zeros(sig.shape[0])
    for ray, start, N in rays_a:
        T = 1.0
        for s in range(start, start + N):
            if T > thr:
                a = 1 - np.exp(-float(sig[s]) * float(deltas[s]))
                w = a * T
                rgb[ray] += w * rgbs[s]
                dep[ray] += w * ts[s]
                op[ray] += w
                ws[s] = w
                T *= 1 - a
    return op, dep, rgb, ws


@pytest.mark.parametrize("dense", [False, True])
def test_composite_fwd_matches_numpy(oracle, dense):
    rng = np.random.default_rng(12)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, dense=dense)
    tot, op, dep, rgb, ws = oracle.composite_train_fwd(sig, rgbs, deltas, ts, rays_a, 1e-4)
    rop, rdep, rrgb, rws = _np_composite(rays_a, sig, rgbs, deltas, ts, 1e-4)
    np.testing.assert_allclose(op, rop, atol=2e-6)
    np.testing.assert_allclose(dep, rdep, atol=2e-6)
    np.testing.assert_allclose(rgb, rrgb, atol=2e-6)
    np.testing.assert_allclose(ws, rws, atol=2e-6)
    if dense:
        assert (tot < rays_a[np.argsort(rays_a[:, 0]), 2]).any()  # early termination exercised


def test_composite_bwd_matches_finite_difference(oracle):
    rng = np.random.default_rng(13)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, n_rays=12, max_n=20)
    deltas = deltas * 30
    n, S = rays_a.shape[0], sig.shape[0]
    go, gd, gr, gw = rng.standard_normal(n), rng.standard_normal(n), rng.standard_normal((n, 3)), rng.standard_normal(S)

    def loss(sig_, rgbs_):
        op, dep, rgb, ws = _np_composite(rays_a, sig_, rgbs_, deltas, ts, 1e-4)
        return (op * go).sum() + (dep * gd).sum() + (rgb * gr).sum() + (ws * gw).sum()

    dsig, drgbs = oracle.composite_train_bwd(go, gd, gr, gw, sig, rgbs, deltas, ts, rays_a, 1e-4)
    eps = 1e-4
    for s in range(0, S, max(1, S // 40)):
        sp, sm = sig.astype(np.float64).copy(), sig.astype(np.float64).copy()
        sp[s] += eps
        sm[s] -= eps
        fd = (loss(sp, rgbs) - loss(sm, rgbs)) / (2 * eps)
        assert abs(fd - dsig[s]) < 1e-4 * max(1.0, abs(fd)), s
        for c in range(3):
            rp, rm = rgbs.astype(np.float64).copy(), rgbs.astype(np.float64).copy()
            rp[s, c] += eps
            rm[s, c] -= eps
            fd = (loss(sig, rp) - loss(sig, rm)) / (2 * eps)
            assert abs(fd - drgbs[s, c]) < 1e-5 * max(1.0, abs(fd))


def test_composite_test_equals_train_when_chunked(oracle):
    """Accumulating chunks with composite_test reproduces the training compositing (no early stop)."""
    rng = np.random.default_rng(14)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, n_rays=40, max_n=50)
    rays_a[:, 0] = np.arange(40)
    tot, op, dep, rgb, ws = oracle.composite_train_fwd(sig, rgbs, deltas, ts, rays_a, 0.0)
    n = 40
    opacity, depth, out = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros((n, 3), np.float32)
    done = np.zeros(n, np.int64)
    chunk = 7
    for it in range(10):
        alive = np.arange(n, dtype=np.int64)
        steps = np.minimum(chunk, rays_a[:, 2] - done)
        pack = np.stack([rays_a[:, 1] + done, steps], 1).astype(np.int64)
        oracle.composite_test(sig, rgbs, deltas, ts, pack, alive, 0.0, opacity, depth, out)
        done += steps
    np.testing.assert_allclose(opacity, op, atol=1e-5)
    np.testing.assert_allclose(out, rgb, atol=1e-5)
    np.testing.assert_allclose(depth, dep, atol=1e-5)


def _reference_test_loop(oracle, model, o, d, esf, thr, max_samples=1024):
    """numpy restatement of the reference's test-time loop (modules/rendering.py:61-158): march <= step samples per
    live ray (raymarching_test resumes at hits_t[:, 0]), shade them, composite_test onto the accumulators, drop the
    rays it marks dead; step = max(min(n_rays // n_alive, 64), min_samples)."""
    n = o.shape[0]
    hits = oracle.ray_aabb_intersect(o, d, model.scale)
    opacity, depth, rgb = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros((n, 3), np.float32)
    alive = np.arange(n, dtype=np.int64)
    samples = total = 0
    min_samples = 1 if esf == 0 else 4
    lo, hi = np.float32(-model.scale), np.float32(model.scale)
    while samples < max_samples and alive.size:
        step = max(min(n // alive.size, 64), min_samples)
        samples += step
        ri, valid, dl, tt, cnt = oracle.raymarching_test(o, d, hits, alive, model.bitfield, model.cascades,
                                                         model.scale, esf, model.grid_size, step)
        v = valid.astype(bool)
        if not v.any():
            break
        ri, dl, tt = ri[v], dl[v], tt[v]
        cnt = cnt.astype(np.int64)
        pack = np.stack([np.cumsum(cnt) - cnt, cnt], 1)
        xyzs = o[ri] + tt[:, None] * d[ri]                       # rendering.py:109-111, fp32
        xn = ((xyzs - lo) / (hi - lo)).astype(np.float32)
        sig, rgbs = oracle.mlp_fwd(oracle.hash_encode_fwd(xn, model.table_for_kernel(), model.layout), d[ri], model.ws)
        oracle.composite_test(sig, rgbs, dl, tt, pack, alive, thr, opacity, depth, rgb)
        alive = alive[alive >= 0]
        total += int(cnt.sum())
    bg = np.float32(1.0 if esf == 0 else 0.0)
    return dict(rgb=rgb + bg * (1 - opacity)[:, None], depth=depth, opacity=opacity, total_samples=total)


@pytest.mark.parametrize("thr", [1e-4, 0.25])
@pytest.mark.parametrize("scene", ["lego", "3casc_esf"])
def test_render_test_equals_reference_loop(oracle, lego_bitfield, rays_factory, scene, thr):
    """oracle render_test (one march of every ray, one composite_test per ray) == the reference's chunked loop on rays
    that stay below max_samples: compositing is sequential per ray and stops at the first sample with T <= threshold,
    however the samples are chunked.  The chunks restart from T = 1 - opacity, hence fp32 rounding, not bits."""
    from oracle.train_step import OracleModel, render_test
    rng = np.random.default_rng(16)
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2)
    table = (rng.uniform(-1, 1, (lay.total_entries, 2)) * 6).astype(np.float32)     # dense-ish medium
    if scene == "lego":
        sc, casc, esf, bits = 0.5, 1, 0.0, lego_bitfield
        o, d = rays_factory(256, seed=16)
    else:
        sc, casc, esf = 2.0, 3, 1 / 256
        bits = (rng.random(casc * 128 ** 3 // 8) < 0.05).astype(np.uint8) * rng.integers(1, 256, casc * 128 ** 3 // 8,
                                                                                          dtype=np.uint8)
        o, d = rays_factory(256, seed=16, radius=1.5)
    ws = _rand_weights(rng)
    ws[1] *= 3                                                                          # larger density logits
    model = OracleModel(lay, table, ws, bits, scale=sc, cascades=casc, half=True)
    got = render_test(model, o, d, esf, thr)
    want = _reference_test_loop(oracle, model, o, d, esf, thr)
    counts = got["rays_a"][:, 2]
    assert counts.max() < 1024 and got["S"] == counts.sum() > 0
    n_term = got["n_term"]
    stopped = n_term < counts                                  # rays whose transmittance fell to the threshold
    assert 0.05 < stopped.mean() < 0.95, stopped.mean()        # both kinds of ray are present
    assert (n_term <= counts).all()
    for k in ("rgb", "depth", "opacity"):
        np.testing.assert_allclose(got[k], want[k], atol=1e-5, err_msg=k)
    # the loop marches whole chunks: at least every sample up to termination, at most every sample
    assert n_term.sum() <= want["total_samples"] <= got["S"]


# ------------------------------------------------------------------------------------------------
def test_packbits_and_morton(oracle):
    rng = np.random.default_rng(15)
    grid = rng.standard_normal(4096).astype(np.float32)
    bits = oracle.packbits(grid, 0.1)
    assert np.array_equal(bits, np.packbits(grid > 0.1, bitorder="little"))
    coords = rng.integers(0, 128, (1000, 3)).astype(np.int32)
    idx = oracle.morton3d(coords)
    assert np.array_equal(oracle.morton3d_invert(idx), coords)
    assert idx.min() >= 0 and idx.max() < 128 ** 3
    assert oracle.morton3d(np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [3, 0, 0]], np.int32)).tolist() == [1, 2, 4, 9]


def test_adam_matches_torch(oracle):
    rng = np.random.default_rng(16)
    n = 1000
    p0 = rng.standard_normal(n).astype(np.float32)
    p = p0.copy()
    m, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
    tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([tp], lr=1e-2, eps=1e-15)
    shadow = np.zeros(n, np.float16)
    for step in range(1, 6):
        g = rng.standard_normal(n).astype(np.float32)
        tp.grad = torch.from_numpy(g.copy())
        opt.step()
        gs = (g * 65536).astype(np.float32)
        oracle.adam_step(p, gs, m, v, 1e-2, step, inv_scale=1.0 / 65536, param_f16=shadow, zero_grad=True)
        assert not gs.any()
    np.testing.assert_allclose(p, tp.detach().numpy(), rtol=1e-5, atol=1e-7)
    assert np.array_equal(shadow, p.astype(np.float16))
    # inf skip
    before = p.copy()
    g = np.full(n, np.inf, np.float32)
    assert oracle.check_finite(g) == 1
    oracle.adam_step(p, g, m, v, 1e-2, 6, found_inf=1)
    assert np.array_equal(p, before)


def test_distortion_matches_numpy_and_fd(oracle):
    rng = np.random.default_rng(17)
    rays_a, sig, rgbs, deltas, ts = _composite_inputs(rng, n_rays=20, max_n=30)
    S = sig.shape[0]
    ws = rng.random(S).astype(np.float32) * 0.1
    # O(n^2) definition of the Mip-NeRF-360 distortion loss on intervals (DVGO-v2 form)
    ref = np.zeros(rays_a.shape[0])
    for ray, start, N in rays_a:
        w, t, d = ws[start:start + N].astype(np.float64), ts[start:start + N].astype(np.float64), deltas[start:start + N]
        # the scan form equals sum_{i>j} 2 w_i w_j (t_i - t_j) + sum_i w_i^2 d_i / 3 for sorted t
        acc = 0.0
        for i in range(N):
            for j in range(i):
                acc += 2 * w[i] * w[j] * (t[i] - t[j])
        ref[ray] = acc + (w * w * d).sum() / 3
    # ts of one ray must be sorted for the identity above: _composite_inputs sorts globally -> sorted per ray
    loss = oracle.distortion_fwd(ws, deltas, ts, rays_a)
    np.testing.assert_allclose(loss, ref, rtol=2e-4, atol=1e-7)
    g = rng.standard_normal(rays_a.shape[0]).astype(np.float32)
    dws = oracle.distortion_bwd(g, ws, deltas, ts, rays_a)
    eps = 1e-3
    for s in range(0, S, max(1, S // 25)):
        wp, wm = ws.copy(), ws.copy()
        wp[s] += eps
        wm[s] -= eps
        fd = ((oracle.distortion_fwd(wp, deltas, ts, rays_a).astype(np.float64) -
               oracle.distortion_fwd(wm, deltas, ts, rays_a)) * g).sum() / (2 * eps)
        assert abs(fd - dws[s]) < 2e-3 * max(1.0, abs(fd)), (s, fd, dws[s])


def test_philox_known_answers(oracle):
    """Random123 kat_vectors for philox4x32 with 10 rounds — pins the generator behind the ray sampler."""
    kat = [
        ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
        ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
        ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
         [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
    ]
    for ctr, key, want in kat:
        got = oracle.philox4x32_10(np.array(ctr, np.uint32), np.array(key, np.uint32))
        assert [int(x) for x in got] == want


def test_sample_ray_batch_matches_dataset_and_get_rays(oracle):
    """Given the reference's own img/pix indices, the sampler equals the gather + get_rays of
    datasets/base.py:53-60 and datasets/ray_utils.py:67-75; its own draws are uniform and step-dependent."""
    from datasets.ray_utils import get_ray_directions, get_rays
    rng = np.random.default_rng(5)
    H = W = 24
    n_img, n = 7, 4096
    K = torch.tensor([[30.0, 0, W / 2], [0, 30.0, H / 2], [0, 0, 1]])
    dirs = get_ray_directions(H, W, K).numpy()
    poses = rng.standard_normal((n_img, 3, 4)).astype(np.float32)
    bank = rng.random((n_img, H * W, 4)).astype(np.float32)   # RGBA bank: only [:, :3] is sampled
    ii = rng.integers(0, n_img, n)
    pi = rng.integers(0, H * W, n)
    got = oracle.sample_ray_batch(bank, poses, dirs, n, img_idxs=ii, pix_idxs=pi)
    ro, rd = get_rays(torch.from_numpy(dirs[pi]), torch.from_numpy(poses[ii]))
    np.testing.assert_array_equal(got["rays_o"], ro.numpy())
    np.testing.assert_allclose(got["rays_d"], rd.numpy(), rtol=1e-6, atol=1e-6)   # torch's sum order is unspecified
    np.testing.assert_array_equal(got["rgb"], bank[ii, pi, :3])
    # own Philox draws: in range, roughly uniform, reproducible, different per step and per seed
    a = oracle.sample_ray_batch(bank, poses, dirs, n, seed=11, step=3)
    b = oracle.sample_ray_batch(bank, poses, dirs, n, seed=11, step=3)
    c = oracle.sample_ray_batch(bank, poses, dirs, n, seed=11, step=4)
    d = oracle.sample_ray_batch(bank, poses, dirs, n, seed=12, step=3)
    assert a["img_idxs"].min() >= 0 and a["img_idxs"].max() == n_img - 1
    assert a["pix_idxs"].min() >= 0 and a["pix_idxs"].max() < H * W
    assert np.array_equal(a["pix_idxs"], b["pix_idxs"]) and np.array_equal(a["noise"], b["noise"])
    assert (a["pix_idxs"] != c["pix_idxs"]).mean() > 0.9 and (a["pix_idxs"] != d["pix_idxs"]).mean() > 0.9
    counts = np.bincount(a["img_idxs"], minlength=n_img)
    assert counts.min() > n / n_img * 0.8
    assert 0.0 <= a["noise"].min() and a["noise"].max() < 1.0 and abs(a["noise"].mean() - 0.5) < 0.02
    np.testing.assert_array_equal(a["rgb"], bank[a["img_idxs"], a["pix_idxs"], :3])
    # 'same_image' strategy (base.py:45-47)
    e = oracle.sample_ray_batch(bank, poses, dirs, 64, fixed_img=2, seed=1)
    assert (e["img_idxs"] == 2).all() and (e["rays_o"] == poses[2, :, 3]).all()


def _closed_form_positions(t0, n, dt):
    """t_{k+1} = fl32(t_k + dt) without the serial chain: inside one binade every step adds the same whole number
    of ulps (dt = sqrt(3)/1024 has an odd mantissa, so the rounding never hits a tie for t >= NEAR_DISTANCE);
    only the step that crosses into the next binade is taken with a real fp32 add."""
    t = np.float32(t0)
    out = [t]
    while len(out) <= n:
        bits = int(t.view(np.uint32))
        e, m = (bits >> 23) & 0xFF, (bits & 0x7FFFFF) | 0x800000
        t1 = np.float32(t + dt)
        b1 = int(t1.view(np.uint32))
        if (b1 >> 23) & 0xFF != e:
            t = t1
            out.append(t)
            continue
        c = ((b1 & 0x7FFFFF) | 0x800000) - m
        j = min(n + 1 - len(out), (0xFFFFFF - m) // c)
        if j == 0:
            t = t1
            out.append(t)
            continue
        ms = m + c * np.arange(1, j + 1, dtype=np.int64)
        out.extend(((e << 23) | (ms & 0x7FFFFF)).astype(np.uint32).view(np.float32))
        t = out[-1]
    return np.array(out[: n + 1], np.float32)


def test_constant_step_recurrence_has_closed_form(oracle, lego_bitfield, rays_factory):
    """Property of the synthetic-scene march (exp_step_factor = 0, ray_march.py:45-74): every sample time of a ray lies
    on ONE occupancy-independent fp32 sequence t_{k+1} = t_k + dt, and that sequence can be generated without the
    serial add chain.  (Basis of the planned cell-stepping march, DESIGN.md §7.)"""
    dt = np.float32(1.7320508075688772 / 1024)
    rng = np.random.default_rng(77)
    for t0 in rng.uniform(0.01, 2.5, 200).astype(np.float32):
        seq = [np.float32(t0)]
        for _ in range(1100):
            seq.append(np.float32(seq[-1] + dt))
        assert np.array_equal(np.array(seq, np.float32).view(np.uint32),
                              _closed_form_positions(t0, 1100, dt).view(np.uint32))
    n = 257
    o, d = rays_factory(n, seed=78)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = rng.random(n, dtype=np.float32)
    ra, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, lego_bitfield, noise, 1, 0.5, 0.0, 128, 1024)
    assert S > 1000
    for r, s0, c in ra:
        if c == 0:
            continue
        t0 = np.float32(hits[r, 0] + np.float32(dt * noise[r]))            # ray_march.py:36-38
        grid = _closed_form_positions(t0, 1100, dt).view(np.uint32)
        assert np.isin(ts[s0:s0 + c].view(np.uint32), grid).all()
        assert (deltas[s0:s0 + c] == dt).all()


@pytest.mark.parametrize("occ", ["lego", "random", "full"])
def test_cellstep_march_equals_reference_march(oracle, lego_bitfield, rays_factory, occ):
    """The cell-stepping loop (closed-form jump over empty cells, one bitfield lookup per cell) emits exactly the
    sample times of the reference-shaped loop — the blueprint for the next marching kernel (DESIGN.md §7)."""
    rng = np.random.default_rng(90)
    n = 1500
    o, d = rays_factory(n, seed=90)
    d[:40] *= -1                                  # rays pointing away / grazing
    bits = {"lego": lego_bitfield, "random": rng.integers(0, 256, 128 ** 3 // 8, dtype=np.uint8),
            "full": np.full(128 ** 3 // 8, 255, np.uint8)}[occ]
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = rng.random(n, dtype=np.float32)
    for max_samples in (1024, 37):
        ra, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, noise, 1, 0.5, 0.0, 128, max_samples)
        ts2, counts, st = oracle.raymarching_cellstep(o, d, hits, bits, noise, 1, 0.5, 128, max_samples, ra, S)
        assert np.array_equal(counts, ra[:, 2])
        assert np.array_equal(ts2.view(np.uint32), ts.view(np.uint32))
    # loop statistics: the inner `while t < t_target` chain is gone (about one real fp32 add per iteration)
    assert st["real_adds"] < 1.1 * st["iterations"] + n


def test_reference_exit_quirk_visits_every_candidate_position(oracle, rays_factory):
    """ray_march.py:66-71 computes the cell exit from the UN-floored grid coordinate, so along an axis with d < 0
    the "exit" is the sample position itself: t_target == t and the loop advances by exactly one step.  Hence, for a
    ray with a negative direction component, the emitted samples are exactly the occupied positions of the
    occupancy-independent t sequence — except inside the outermost half cell, where the coordinate is clamped to
    grid_size - 1 and a real multi-step jump happens.  (Why empty-space skipping buys the reference nothing, and
    the basis of the independent-positions marching fast path planned in DESIGN.md §7.)"""
    f32 = np.float32
    rng = np.random.default_rng(3)
    n = 1200
    o, d = rays_factory(n, seed=11)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = rng.random(n, dtype=np.float32)
    bits = rng.integers(0, 256, 128 ** 3 // 8, dtype=np.uint8)
    full = np.full(128 ** 3 // 8, 255, np.uint8)
    ra_f, x_f, _, _, ts_f, _ = oracle.raymarching_train(o, d, hits, full, noise, 1, 0.5, 0.0, 128, 4096)   # every position
    ra, _, _, _, ts, _ = oracle.raymarching_train(o, d, hits, bits, noise, 1, 0.5, 0.0, 128, 4096)
    v = (f32(0.5) * (x_f * f32(2.0) + f32(1.0))).astype(np.float32) * f32(128.0)       # utils/ray_march grid coordinate
    v = np.minimum(np.maximum(v, f32(0)), f32(127)).astype(np.float32)
    idx = oracle.morton3d(v.astype(np.int32)).astype(np.int64)
    occ = ((bits[idx >> 3] >> (idx & 7)) & 1).astype(bool)
    checked = 0
    for r in range(n):
        if d[r].min() > -1e-3:
            continue
        s0, c = ra_f[r, 1], ra_f[r, 2]
        emitted = np.isin(ts_f[s0:s0 + c].view(np.uint32), ts[ra[r, 1]:ra[r, 1] + ra[r, 2]].view(np.uint32))
        differ = emitted != occ[s0:s0 + c]
        assert not emitted[~occ[s0:s0 + c]].any()                               # nothing is emitted from an empty cell
        assert (v[s0:s0 + c][differ] == 127.0).any(axis=1).all()                # skipped positions: clamped layer only
        checked += 1
    assert checked > n // 2


def test_chunked_fast_path_emulation_equals_reference_march(oracle, lego_bitfield, rays_factory):
    """Lane-level emulation of the planned warp kernel: chunks whose empty lanes all have a negative, unclamped axis
    take the independent-positions path (emit = occupied lanes), the rest the sequential loop — same sample times,
    and the fast path covers the bulk of the chunks."""
    rng = np.random.default_rng(91)
    n = 2500
    o, d = rays_factory(n, seed=91)
    d[:200] = np.abs(d[:200])                     # all-positive directions: the only rays with real jumps
    d[200:240, 2] = 0.0                           # axis-parallel components (1/d = inf)
    hits = oracle.ray_aabb_intersect(o, d, 0.5)
    noise = rng.random(n, dtype=np.float32)
    for bits in (lego_bitfield, rng.integers(0, 256, 128 ** 3 // 8, dtype=np.uint8)):
        for max_samples in (1024, 50):
            ra, _, _, _, ts, S = oracle.raymarching_train(o, d, hits, bits, noise, 1, 0.5, 0.0, 128, max_samples)
            ts2, counts, st = oracle.raymarching_lanes(o, d, hits, bits, noise, 0.5, 128, max_samples, ra, S)
            assert np.array_equal(counts, ra[:, 2])
            assert np.array_equal(ts2.view(np.uint32), ts.view(np.uint32))
            assert st["regular_chunks"] > 8 * st["general_chunks"]


# ---- fast_hash / under_hash known-answer test (Python-int arithmetic, tests/hash_kat.py) -------------------
@pytest.mark.parametrize("max_res", [1024, 4096])
def test_hash_index_known_answers(oracle, max_res):
    """The oracle's corner indices / weights against hash_encoder.py:43-71,108-139 evaluated with Python integers:
    a table that stores its own entry index makes the encoder output reveal every index it touched."""
    import hash_kat as K
    from taichi_nerfs_b200.layout import make_hash_layout
    lay = make_hash_layout(2 ** 19, 16, 16, max_res, 2)
    if max_res == 1024:
        for p, level, corner, entry in K.hand_computed_vectors():
            assert K.corner_table(lay, p, level)[corner][0] == entry
    table = K.index_table(lay)
    want = K.expected(lay, K.POINTS)
    got = oracle.hash_encode_fwd(K.POINTS, table.reshape(-1), lay).astype(np.float64)
    # outputs are O(index) ~ 5e6; a wrong index is off by >= 1 * weight, fp32 summation slack is ~1e-7 relative
    np.testing.assert_allclose(got, want, rtol=2e-6, atol=0.5)
