"""Test-time frames against the CPU oracle: the compositing kernel of the compacting renderer on synthetic rounds, and
whole frames of FrameRenderer (render(test_time=True) of the stock model) and of the non-compacting render_frame
against oracle.train_step.render_test (march every ray with max_samples per ray, shade, composite each ray once)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle.train_step import OracleModel, make_rays, render_test

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

DEV = "cuda"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def _ptr(t):
    return C.c_void_p(t.data_ptr())


# ---- composite_round against oracle.composite_test ----------------------------------------------------------------
def _lanes(limit):
    return 4 if limit <= 4 else 8 if limit <= 8 else 16 if limit <= 16 else 32     # ngp_composite_round's choice


def _round_inputs(rng, n_rays, n_alive, limit, half):
    """One synthetic round: a live list (a permutation of a subset of the rays), per-slot sample counts up to the round
    limit in a shuffled row layout, non-zero starting accumulators, and rays of every kind the kernel must tell apart."""
    G = _lanes(limit)
    alive = rng.permutation(n_rays)[:n_alive].astype(np.int32)
    cnt = rng.integers(0, limit + 1, n_alive)
    kind = np.arange(n_alive) % 8
    # 0/1: random medium (light or dense), 2: no samples, march finished (t_cur = +inf), 3: leaves the box this round,
    # 4: opaque first sample, 5/6: opaque sample on either side of the first group boundary, 7: opaque last sample
    cnt[kind == 2] = 0               # (with t_cur = +inf, as every ray the round march gives no sample)
    cnt[(kind >= 4) & (cnt == 0)] = 1
    if limit > G:
        cnt[(kind == 5) | (kind == 6)] = np.maximum(cnt[(kind == 5) | (kind == 6)], G + 1)
    S = int(cnt.sum())
    order = rng.permutation(n_alive)                  # rows are reserved in atomic order, not slot order
    start = np.empty(n_alive, np.int64)
    start[order] = np.cumsum(cnt[order]) - cnt[order]
    rays_a = np.stack([alive, start, cnt], 1).astype(np.int32)
    deltas = (1.7320508075688772 / 1024 * rng.uniform(1, 20, S)).astype(np.float32)
    dense = np.repeat(kind == 1, cnt)
    sig = (rng.random(S) * np.where(dense, 300.0, 3.0)).astype(np.float32)
    for k, pos in ((4, lambda c: 0), (5, lambda c: min(G - 1, c - 1)), (6, lambda c: min(G, c - 1)), (7, lambda c: c - 1)):
        sel = np.nonzero(kind == k)[0]
        sig[start[sel] + np.array([pos(c) for c in cnt[sel]], np.int64)] = 1e5      # alpha == 1: T drops to 0 here
    rgbs = rng.random((S, 3)).astype(np.float16 if half else np.float32)
    ts = (rng.random(S) * 2).astype(np.float32)
    hits = np.stack([np.full(n_rays, 0.05), rng.uniform(1.0, 3.0, n_rays)], 1).astype(np.float32)
    t_cur = (hits[:, 1] * rng.uniform(0.1, 0.9, n_rays)).astype(np.float32)
    t_cur[alive[cnt == 0]] = np.inf
    t_cur[alive[kind == 3]] = hits[alive[kind == 3], 1] * np.float32(rng.choice([1.0, 1.5]))
    opacity = (rng.random(n_rays) * 0.5).astype(np.float32)
    depth = (rng.random(n_rays) * 0.5).astype(np.float32)
    rgb = (rng.random((n_rays, 3)) * 0.5).astype(np.float32)
    return rays_a, sig, rgbs, deltas, ts, hits, t_cur, opacity, depth, rgb


def _near_threshold(rays_a, sig, deltas, opacity, thr):
    """Slots where the fp64 transmittance before some sample lies within 1e-5 relative of the threshold: there the group
    prefix products may end the ray one sample before or after the oracle's sequential product."""
    out = np.zeros(rays_a.shape[0], bool)
    for i, (ray, s0, c) in enumerate(rays_a):
        if c:
            a = np.exp(-sig[s0:s0 + c].astype(np.float64) * deltas[s0:s0 + c].astype(np.float64))
            Tb = (1.0 - np.float64(opacity[ray])) * np.concatenate([[1.0], np.cumprod(a)[:-1]])
            out[i] = (np.abs(Tb - thr) <= 1e-5 * thr).any()
    return out


def _run_composite_round(oracle, n_rays, n_alive, limit, half, thr, seed):
    from taichi_nerfs_b200 import _lib
    rng = np.random.default_rng(seed)
    rays_a, sig, rgbs, deltas, ts, hits, t_cur, op0, dep0, rgb0 = _round_inputs(rng, n_rays, n_alive, limit, half)
    # oracle: one composite_test call over the round's samples of every live ray
    r_alive = rays_a[:, 0].astype(np.int64)
    r_op, r_dep, r_rgb = op0.copy(), dep0.copy(), rgb0.copy()
    oracle.composite_test(sig, rgbs, deltas, ts, rays_a[:, 1:].astype(np.int64), r_alive, thr, r_op, r_dep, r_rgb)
    want = set(int(r) for r in r_alive[r_alive >= 0] if t_cur[r] < hits[r, 1])
    # kernel
    state = torch.zeros(8, device=DEV, dtype=torch.int32)
    state[2] = n_alive
    g_op, g_dep, g_rgb = T(op0), T(dep0), T(rgb0)
    nxt = torch.full((n_rays,), -7, device=DEV, dtype=torch.int32)
    t_sig, t_rgbs, t_dl, t_ts, t_ra, t_hits, t_tc = T(sig), T(rgbs), T(deltas), T(ts), T(rays_a), T(hits), T(t_cur)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.load().ngp_composite_round(_ptr(t_sig), _ptr(t_rgbs), 1 if half else 0, _ptr(t_dl), _ptr(t_ts),
                                               _ptr(t_ra), _ptr(state), _ptr(t_tc), _ptr(t_hits), thr, _ptr(g_op),
                                               _ptr(g_dep), _ptr(g_rgb), _ptr(nxt), n_rays, limit, st))
    g_op, g_dep, g_rgb, state, nxt = N(g_op), N(g_dep), N(g_rgb), N(state), N(nxt)
    amb = _near_threshold(rays_a, sig, deltas, op0, thr)
    assert amb.mean() < 0.01, amb.mean()
    ok = np.ones(n_rays, bool)
    ok[rays_a[amb, 0]] = False
    # group prefix products are not sequential products: 2e-5 absolute, as test_composite_train_fwd_bwd
    err = max(np.abs(g_op - r_op)[ok].max(), np.abs(g_dep - r_dep)[ok].max(), np.abs(g_rgb - r_rgb)[ok].max())
    assert err <= 2e-5, err
    # rays that are not on the live list are left alone
    off = np.ones(n_rays, bool)
    off[rays_a[:, 0]] = False
    assert np.array_equal(g_op[off], op0[off]) and np.array_equal(g_rgb[off], rgb0[off])
    # the next live list: no duplicates, exactly the rays with T > threshold that are still inside the box
    n_next = int(state[3])
    got = nxt[:n_next]
    assert len(set(got.tolist())) == n_next
    assert (nxt[n_next:] == -7).all()
    amb_rays = set(int(r) for r in rays_a[amb, 0])
    assert set(got.tolist()) - amb_rays == want - amb_rays
    return err, n_next


@pytest.mark.parametrize("thr", [1e-4, 0.25])
@pytest.mark.parametrize("half", [True, False], ids=["f16", "f32"])
@pytest.mark.parametrize("limit", [1, 4, 5, 8, 9, 16, 17, 32, 33, 512])
def test_composite_round_matches_oracle(oracle, limit, half, thr):
    """Every lane-group width (4/8/16/32 lanes per ray) and the multi-chunk loop, against composite_test."""
    n_alive = 3000 if limit < 512 else 1500
    _run_composite_round(oracle, 4 * n_alive + 11, n_alive, limit, half, thr, seed=limit)


@pytest.mark.parametrize("limit", [4, 32])
def test_composite_round_more_rays_than_one_wave(oracle, limit):
    """More live rays than the persistent grid covers in one pass (8 CTAs per SM, 8 warps, 32 / G rays per warp)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_alive = 8 * sms * 8 * (32 // _lanes(limit)) * 2 + 123
    _run_composite_round(oracle, n_alive + 1000, n_alive, limit, True, 1e-4, seed=100 + limit)


# ---- whole frames against oracle.train_step.render_test ----------------------------------------------------------
def _weights(rng):
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    ws = [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]
    ws[1] *= 3                                                               # larger density logits
    return ws


def _models(scale, max_res, half, bits, seed, table_amp=6.0, fog=False):
    """The same parameters as an NGP on the GPU and as an OracleModel (the fp16 shadow of half models is the table the
    kernels read, exported with table_f16(), so both sides encode identical tables)."""
    from modules.networks import NGP
    from taichi_nerfs_b200.fused_mlp import mlp_weights
    rng = np.random.default_rng(seed)
    m = NGP(scale=scale, max_res=max_res, half_opt=half).to(DEV)
    enc = m.pos_encoder
    table = (rng.uniform(-1, 1, tuple(enc.hash_table.shape)) * table_amp).astype(np.float32)
    ws = _weights(rng)
    if fog:
        ws[1][0] = 0.0                    # density logit 0 everywhere: sigma = exp(0) = 1
    with torch.no_grad():
        enc.hash_table.copy_(T(table))
        for p, w in zip(mlp_weights(m), ws):
            p.copy_(T(w))
        m.density_bitfield.copy_(T(bits))
    om = OracleModel(enc._layout, table, ws, bits, scale, m.cascades, m.grid_size, half)
    if half:
        om.shadow = N(enc.table_f16()).reshape(-1)
        assert np.array_equal(om.shadow, table.reshape(-1).astype(np.float16))
    return m, om


def _flip_weight(ref, thr):
    """Per ray: the weight a termination flip can move.  A sample is composited while the transmittance before it is
    above the threshold; the kernels' sigma differs from the oracle's by ~1e-3 relative, so T differs by ~1e-3 * -ln T.
    Where the fp64 T before the last composited sample, or before the first one left out, lies that close to the
    threshold, the GPU may stop one sample earlier or later, which moves alpha * T ~ alpha * threshold of weight."""
    ra, n_term = ref["rays_a"].astype(np.int64), ref["n_term"].astype(np.int64)
    x = ref["sigmas"].astype(np.float64) * ref["deltas"].astype(np.float64)
    cs = np.concatenate([[0.0], np.cumsum(x)])
    rel = 3e-3 * max(1.0, -np.log(thr))
    w = np.zeros(ra.shape[0])
    for k in (n_term - 1, n_term):
        valid = (k >= 0) & (k < ra[:, 2])
        s = np.minimum(ra[:, 1] + np.maximum(k, 0), x.size - 1)
        Tb = np.exp(-(cs[s] - cs[ra[:, 1]]))
        near = valid & (np.abs(Tb / thr - 1.0) <= rel)
        w = np.maximum(w, np.where(near, -np.expm1(-x[s]) * Tb, 0.0))
    return w


def _check_frame(out, ref, hits, thr, what):
    """Per-ray tolerances from the MLP error model (sigma within ~1e-3 relative, fp16 rgb within 2e-3), plus, on the
    few rays whose termination may flip, the weight the flip moves.  Returns the measured maxima."""
    op, dep, rgb = N(out["opacity"]), N(out["depth"]), N(out["rgb"])
    t_max = float(hits[:, 1].max())
    flip = _flip_weight(ref, thr)
    e_op = np.abs(op - ref["opacity"])
    e_rgb = np.abs(rgb - ref["rgb"]).max(1)
    e_dep = np.abs(dep - ref["depth"]) / t_max
    e = dict(opacity=float(e_op.max()), rgb=float(e_rgb.max()), depth=float(e_dep.max()),
             flip_rays=int((flip > 0).sum()))
    print(what, "max errors", e, "samples", int(out["total_samples"]), "oracle S", ref["S"],
          "to termination", int(ref["n_term"].sum()))
    # measured on an H100 (400 W): opacity <= 4.7e-4, rgb <= 4.9e-4, depth <= 3.2e-4 * t_max at threshold 1e-4 (Lego,
    # fp16 and fp32 encoder, garden, fog).  At threshold 0.25: opacity 1.02e-3, depth 6.4e-4 * t_max, on a ray that is
    # not near a termination flip.  A sigma error moves the opacity by T_end * sum(d sigma * delta): rays stopped at 0.25
    # end with ~2500x the transmittance of rays stopped at 1e-4, and the fp16 density logit gives sigma more than 1e-3
    # relative error where the logit is large, hence the wider opacity bound there
    op_bound = 1e-3 if thr <= 1e-3 else 2e-3
    assert (flip > 1e-4).mean() < 0.01, (what, e)          # flips that move more than 1e-4 of weight are rare
    assert (e_op - flip).max() <= op_bound, (what, e)
    assert (e_rgb - flip).max() <= 3e-3, (what, e)
    assert (e_dep - flip).max() <= 1e-3, (what, e)
    # samples shaded: at least every sample up to termination, at most every sample the capped march has
    assert int(ref["n_term"].sum()) <= int(out["total_samples"]) <= ref["S"], what
    return e


LEGO = dict(scale=0.5, max_res=1024, esf=0.0, n=20000, radius=1.4)
GARDEN = dict(scale=16.0, max_res=4096, esf=1 / 256, n=1200, radius=3.0)


def _case(name, half=True):
    if name == "lego":
        cfg = LEGO
        bits = np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"].copy()
    else:
        cfg = GARDEN
        bits = np.random.default_rng(5).integers(0, 256, 6 * 128 ** 3 // 8, dtype=np.uint8)
    m, om = _models(cfg["scale"], cfg["max_res"], half, bits, seed=11)
    o, d = make_rays(cfg["n"], seed=12, radius=cfg["radius"])
    return cfg, m, om, o, d


def _render(m, o, d, esf, thr):
    import modules.rendering as R
    with torch.autocast("cuda", dtype=torch.float16):
        return R.render(m, T(o), T(d), test_time=True, exp_step_factor=esf, T_threshold=thr)


def _frame_vs_oracle(name, half, thr):
    from oracle import oracle as O
    from taichi_nerfs_b200.render_frame import FrameRenderer
    cfg, m, om, o, d = _case(name, half)
    ref = render_test(om, o, d, cfg["esf"], thr)
    hits = O.ray_aabb_intersect(o, d, cfg["scale"])
    out = _render(m, o, d, cfg["esf"], thr)
    assert (o.shape[0], float(cfg["esf"]), float(thr), T(o).device) in m._frame_renderers   # the compacting renderer
    _check_frame(out, ref, hits, thr, f"{name} half={half} thr={thr}")
    # graph replay == eager enqueue, bit for bit (per-ray results do not depend on row order)
    again = _render(m, o, d, cfg["esf"], thr)
    eager = FrameRenderer(m, o.shape[0], cfg["esf"], thr, use_graph=False).render(T(o), T(d))
    for k in ("opacity", "depth", "rgb", "total_samples"):
        assert torch.equal(out[k], again[k]) and torch.equal(out[k], eager[k]), k
    if ref["n_term"].sum() < ref["S"]:
        assert (ref["n_term"] < ref["rays_a"][:, 2]).mean() > 0.02        # early termination is exercised
    return m, om, o, d, ref, hits


@pytest.mark.parametrize("thr", [1e-4, 0.25])
def test_frame_lego_f16(oracle, thr):
    _frame_vs_oracle("lego", True, thr)


def test_frame_lego_f32_encoder(oracle):
    """fp32 hash table: fp32 embeddings into the MLP kernel."""
    _frame_vs_oracle("lego", False, 1e-4)


def test_frame_garden(oracle):
    """scale 16, 6 cascades, max_res 4096, exp_step_factor 1/256 (background 0), random occupancy, rays inside the box."""
    _frame_vs_oracle("garden", True, 1e-4)


def test_frame_fog_stops_at_max_samples(oracle):
    """sigma = 1 everywhere, every cell occupied, no ray terminates: the rays outlast the scheduled rounds and take the
    host-driven extra rounds, which must stop every ray at max_samples samples like the one-shot march."""
    from oracle import oracle as O
    from taichi_nerfs_b200.render_frame import FrameRenderer
    cfg = dict(GARDEN, n=1000)
    bits = np.full(6 * 128 ** 3 // 8, 255, np.uint8)
    m, om = _models(cfg["scale"], cfg["max_res"], True, bits, seed=13, fog=True)
    o, d = make_rays(cfg["n"], seed=14, radius=cfg["radius"])
    thr = 1e-30
    ref = render_test(om, o, d, cfg["esf"], thr)
    assert (ref["rays_a"][:, 2] == 1024).all() and (ref["n_term"] == 1024).all()
    fr = FrameRenderer(m, cfg["n"], cfg["esf"], thr)
    out = fr.render(T(o), T(d))
    assert fr.rounds_run > len(FrameRenderer.SCHEDULE)
    assert int(out["total_samples"]) == ref["S"], (int(out["total_samples"]), ref["S"])
    _check_frame(out, ref, O.ray_aabb_intersect(o, d, cfg["scale"]), thr, "fog")


# ---- the non-compacting render_frame ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lego", "garden"])
def test_render_frame_passes_match_oracle(oracle, monkeypatch, name):
    """render_frame (the path of models the compacting renderer does not take): the first frame marches in two passes
    and learns the row capacity, the second takes the single-pass march; then a frame that needs more rows than were
    learned overflows the single-pass buffers (dropped > 0) and is rendered again by the two-pass march."""
    from oracle import oracle as O
    from taichi_nerfs_b200 import render_frame as RF
    calls = dict(count=0, frame=0)
    real_count, real_frame = RF.ops.raymarching_train_count, RF.ops.raymarching_frame

    def count(*a, **k):
        calls["count"] += 1
        return real_count(*a, **k)

    def frame(*a, **k):
        calls["frame"] += 1
        out = real_frame(*a, **k)
        calls["dropped"] = int(a[9][1])                # counter = (rows requested, rays dropped)
        return out
    monkeypatch.setattr(RF.ops, "raymarching_train_count", count)
    monkeypatch.setattr(RF.ops, "raymarching_frame", frame)
    cfg, m, om, o, d = _case(name)
    thr = 1e-4

    def render_frame(o, d):
        with torch.autocast("cuda", dtype=torch.float16):
            return RF.render_frame(m, T(o), T(d), cfg["esf"], thr)
    ref = render_test(om, o, d, cfg["esf"], thr)
    hits = O.ray_aabb_intersect(o, d, cfg["scale"])
    first = render_frame(o, d)
    assert calls == dict(count=1, frame=0)
    second = render_frame(o, d)
    assert calls["count"] == 1 and calls["frame"] == 1 and calls["dropped"] == 0
    for out, what in ((first, "two-pass"), (second, "single-pass")):
        _check_frame(out, ref, hits, thr, f"render_frame {name} {what}")
        # every marched sample is shaded
        assert int(out["total_samples"]) == ref["S"]
    for k in ("opacity", "depth", "rgb"):
        assert torch.equal(first[k], second[k]), k
    # learned capacity from a frame that misses the scene, then a frame that needs more rows
    m.__dict__.pop("_frame_capacity", None)
    away = o * 40.0                                         # far outside the box, looking away from it
    empty = render_frame(away, -d)
    assert int(empty["total_samples"]) == 0
    assert ref["S"] > 1 << 16
    calls.update(count=0, frame=0)
    third = render_frame(o, d)
    assert calls["frame"] == 1 and calls["dropped"] > 0 and calls["count"] == 1      # overflow -> two-pass march
    for k in ("opacity", "depth", "rgb", "total_samples"):
        assert torch.equal(third[k], first[k]), k
