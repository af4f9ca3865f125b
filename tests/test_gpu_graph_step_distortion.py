"""The distortion loss in the graph-captured training step: ngp_ray_head_fused_distortion (one launch, one warp per
ray: composite forward + background + MSE + distortion loss + composite backward with the distortion's dL/dw) and
StaticTrainStep(distortion_loss_w=...).

- fp64 distortion reference (`np_distortion_f64`) against the oracle's distortion_fwd/bwd and central differences (CPU);
- the head comparator `check_head_dist` against the fp64 reference, fed the fp64 result rounded to fp32 (accepted) and
  with each fault a looser check lets through (rejected) (CPU);
- the kernel against fp64 on synthetic rays: fp16 / fp32 colours, thresholds 1e-4 and 0.25, 0 .. 5000 samples per ray
  (past the 4096 whose chunk-start carries stay in shared memory), constant and exp_step_factor 1/256 deltas,
  w_d in {1e-3, 1e-2, 1};
- the kernel against the module path's kernel chain on a real march, and with w_d = 0 against ngp_ray_head_fused;
- the step against NGPTrainer.step(extra_loss=w_d * distortion_loss(res).mean()), eager and graph, sync and overlap;
- the head stage on the step's own buffers (Lego bitfield, garden config) against fp64;
- train.py --graph_step --distortion_loss_w 1e-2 on the analytic scene.

Loss:  loss_ray = sum_k w_k (2 (t_k W_<k - WT_<k) + w_k delta_k / 3)  (W, WT: sums of w and w t over the ray), and
dL/dw_k = 2 (t_k W_<k - WT_<k) + 2 (WT_>k - t_k W_>k) + 2/3 w_k delta_k (Mip-NeRF 360, modules/distortion.py).
"""
import ctypes as C

import numpy as np
import pytest

from composite_ref import U, _check_composite_bwd, kernel_termination, np_composite_f64, termination_window

DEV = "cuda"
F32, F16 = 0, 1


# ---- fp64 references ---------------------------------------------------------------------------------------------------
def np_distortion_f64(w, deltas, ts, rays_a, faults=()):
    """Per ray (indexed by ray id): loss_ray and its sum of |terms|; per sample: dloss_ray/dw and its sum of |terms|.
    `faults` restates the formula wrongly (for the comparator tests): "no_w2d" drops w^2 delta / 3, "sel0" gives the
    first sample the selector t_0 w_0, "self_suffix" lets the suffix W_>k include the sample itself (in both W_>k and
    WT_>k its terms w_k t_k - t_k w_k cancel exactly, so only a one-sided slip changes dL/dw)."""
    n, S = rays_a.shape[0], w.size
    loss, lmag = np.zeros(n), np.zeros(n)
    grad, gmag = np.zeros(S), np.zeros(S)
    for r, s0, cnt in rays_a:
        if cnt == 0:
            continue
        sl = slice(s0, s0 + cnt)
        wk, t, d = w[sl].astype(np.float64), ts[sl].astype(np.float64), deltas[sl].astype(np.float64)
        wt = wk * t
        Wp = np.concatenate([[0.0], np.cumsum(wk)[:-1]])            # W_<k
        WTp = np.concatenate([[0.0], np.cumsum(wt)[:-1]])           # WT_<k
        Ws = np.concatenate([np.cumsum(wk[::-1])[::-1][1:], [0.0]])  # W_>k
        WTs = np.concatenate([np.cumsum(wt[::-1])[::-1][1:], [0.0]])
        if "self_suffix" in faults:
            Ws = Ws + wk
        sel = t * Wp - WTp
        if "sel0" in faults:
            sel[0] = t[0] * wk[0]
        w2d = 0.0 if "no_w2d" in faults else 1.0
        loss[r] = (wk * (2 * sel + w2d * wk * d / 3)).sum()
        lmag[r] = (wk * (2 * (t * Wp + WTp) + wk * d / 3)).sum()
        grad[sl] = 2 * sel + 2 * (WTs - t * Ws) + w2d * 2 / 3 * wk * d
        gmag[sl] = 2 * (t * Wp + WTp) + 2 * (WTs + t * Ws) + 2 / 3 * wk * d
    return loss, lmag, grad, gmag


def head_ref(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, thr, n_active=None, faults=()):
    """fp64 head with the distortion loss.  Faults (comparator tests): those of np_distortion_f64, "no_gw" (dL/dw not
    passed through the compositing) and "coef_n" (coefficient scale w_d instead of scale w_d / n_rays)."""
    n, S = rays_a.shape[0], sig.size
    z, zs = np.zeros(n), np.zeros(S)
    fwd = np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, z, z, np.zeros((n, 3)), zs, n_active=n_active)
    out = fwd["rgb"] + bg * (1 - fwd["op"])[:, None]
    dd = out - gt.astype(np.float64)
    g = scale * 2 * dd / (3 * n)
    go = -bg * g.sum(1)
    loss_ray, lmag, dw, gmag = np_distortion_f64(fwd["w"], deltas, ts, rays_a, faults)
    coef_d = scale * w_d / (1 if "coef_n" in faults else n)
    gw = np.zeros(S) if "no_gw" in faults else coef_d * dw
    ref = np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, z, g, gw, n_active=n_active)
    # the same compositing with |dL/dw| replaced by its sum of |terms|: ref["mag"] for the tolerance (see check_head_dist)
    ref["mag"] = np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, z, g, scale * w_d / n * gmag,
                                  n_active=n_active)["mag"]
    loss = (dd ** 2).sum() + 3 * w_d * loss_ray.sum()
    return dict(fwd=fwd, out=out, dd=dd, ref=ref, loss=loss, loss_ray=loss_ray, lmag=lmag, gw=gw)


def check_head_dist(got, sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, thr, half, what, faults=()):
    """Comparator of one head launch: got = (loss_sum, opacity, rgb, dsig, drgbs) as numpy.  The termination index of
    every ray is the kernel's own, accepted only inside the fp32 window of the threshold (tests/composite_ref.py).

    Error bound of the distortion term.  The kernel's w_k carries the compositing's relative error (the conditioning
    factor k = N + 4 / min a of np_composite_f64 bounds it by a few k u).  Its W_<k, WT_<k, W_>k, WT_>k are fp32 sums
    of non-negative terms: within-warp tree (5 roundings) plus one carry per chunk (N / 32), so each is off by at most
    (N / 32 + 6) u of itself.  The products and the final sum of dL/dw_k add < 8 u.  So |dL/dw_k - exact| <=
    2 k u * coef_d * gmag_k, gmag_k the sum of |terms| of dL/dw_k.  dL/dw_k enters dL/dsigma_s = delta_s (T_{s+1} G_s -
    sum_{j>s} w_j G_j) linearly, so the compositing bound 8 k u * mag_s holds with |dL/dw| in mag replaced by
    coef_d * gmag (head_ref's ref["mag"]).  loss_ray: sign-coherent sum of w-weighted terms, off by <= 8 k u lmag."""
    ls, op, rgb, dsig, drgbs = got
    n_lo, n_hi, n64 = termination_window(sig, deltas, rays_a, thr)
    n_k = kernel_termination(dsig, drgbs, rays_a)
    bad = np.flatnonzero((n_k < n_lo) | (n_k > n_hi))
    assert bad.size == 0, f"{what}: {bad.size} rays stop outside the fp32 window of the threshold"
    h = head_ref(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, thr, n_active=n_k, faults=faults)
    fwd, out, dd, ref = h["fwd"], h["out"], h["dd"], h["ref"]
    _check_composite_bwd(dsig, drgbs, ref, half, what)
    k = fwd["kray"]
    assert (np.abs(op - fwd["op"]) <= 8 * k * U * fwd["op"] + 1e-30).all(), f"{what}: opacity"
    e_out = 8 * k[:, None] * U * (np.abs(out) + 2)
    assert (np.abs(rgb - out) <= e_out).all(), f"{what}: rgb"
    # mse part as check_head of tests/test_gpu_graph_step_grads.py, plus 3 w_d * 8 k u lmag per ray and the atomic sum
    tol = ((2 * np.abs(dd) * e_out).sum() + 3 * w_d * (8 * k * U * h["lmag"]).sum()
           + 16 * rays_a.shape[0] * U * ((dd ** 2).sum() + 3 * w_d * h["lmag"].sum()))
    assert abs(float(np.ravel(ls)[0]) - h["loss"]) <= tol, f"{what}: loss_sum {np.ravel(ls)[0]} vs {h['loss']} (tol {tol:.3e})"
    return h


# ---- CPU: the reference and the comparator ---------------------------------------------------------------------------
def _rays(rng, counts, esf, x_lo=0.01, x_hi=0.3, wall=None, long_x=(0.5e-4, 1.5e-4), d_const=1.7e-3):
    """Rays of the given sample counts.  x = sigma delta per sample: [x_lo, x_hi) on rays under 1000 samples, long_x on
    longer ones; `wall` = {ray: sample} puts a dense sample (x = 30) there.  Deltas constant (esf 0) or growing as
    t / 256 (the exp_step_factor marching of large scenes), ts the interval midpoints."""
    sd, dl, tt = [], [], []
    for r, c in enumerate(counts):
        x = rng.uniform(*(long_x if c >= 1000 else (x_lo, x_hi)), c)
        if wall and r in wall:
            x[wall[r]] = 30.0
        t0 = rng.uniform(0.05, 0.5)
        if esf == 0:
            d = np.full(c, d_const)
        else:
            d = np.empty(c)
            t = t0
            for i in range(c):
                d[i] = min(max(t * esf, 1.7e-3), 0.1)
                t += d[i]
        sd.append(x)
        dl.append(d)
        tt.append(t0 + np.cumsum(d) - d / 2)
    sd, deltas, ts = np.concatenate(sd), np.concatenate(dl).astype(np.float32), np.concatenate(tt).astype(np.float32)
    sig = (sd / deltas).astype(np.float32)
    counts = np.array(counts)
    n = counts.size
    rays_a = np.stack([rng.permutation(n), np.cumsum(counts) - counts, counts], 1).astype(np.int32)
    return rays_a, sig, deltas, ts


def test_distortion_reference_matches_oracle_and_central_differences(oracle):
    rng = np.random.default_rng(3)
    counts = [0, 1, 5, 31, 32, 33, 70, 200]
    rays_a = np.stack([rng.permutation(len(counts)), np.cumsum(counts) - counts, counts], 1).astype(np.int32)
    S = int(np.sum(counts))
    ws = rng.uniform(0, 0.05, S).astype(np.float32)
    deltas = rng.uniform(1e-3, 2e-2, S).astype(np.float32)
    ts = np.zeros(S, np.float32)
    for r, s0, c in rays_a:
        ts[s0:s0 + c] = 0.2 + np.cumsum(deltas[s0:s0 + c]) - deltas[s0:s0 + c] / 2
    loss, lmag, grad, gmag = np_distortion_f64(ws, deltas, ts, rays_a)
    # oracle (fp32, sequential): within its own rounding of the sums of |terms|
    lo = oracle.distortion_fwd(ws, deltas, ts, rays_a)
    assert (np.abs(lo - loss) <= 8 * max(counts) * U * lmag + 1e-30).all()
    gref = oracle.distortion_bwd(np.ones(len(counts), np.float32), ws, deltas, ts, rays_a)
    assert (np.abs(gref - grad) <= 8 * max(counts) * U * gmag).all()
    # central differences of the fp64 loss (quadratic in w: exact up to rounding)
    w64 = ws.astype(np.float64)
    for s in rng.choice(S, 40, replace=False):
        e = np.zeros(S)
        e[s] = 1e-4
        up = np_distortion_f64(w64 + e, deltas, ts, rays_a)[0].sum()
        dn = np_distortion_f64(w64 - e, deltas, ts, rays_a)[0].sum()
        assert abs((up - dn) / 2e-4 - grad[s]) <= 1e-8 * max(gmag[s], 1.0), s


def _cpu_case(half, esf=0.0):
    """Short rays of coarse samples (delta 0.05) with large weights: there the w^2 delta / 3 term and the first
    sample's selector are a visible part of dL/dw, as they are on the coarse far samples of a large scene."""
    rng = np.random.default_rng(11 + half)
    rays_a, sig, deltas, ts = _rays(rng, [0, 1, 2, 5, 7, 12, 31, 33, 40], esf, x_lo=0.05, x_hi=0.4, d_const=0.05)
    n, S = rays_a.shape[0], sig.size
    rgbs = (rng.random((S, 3)) * 0.8 + 0.1).astype(np.float16 if half else np.float32)
    gt = rng.random((n, 3)).astype(np.float32)
    return sig, rgbs, deltas, ts, rays_a, gt


def _emulated(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, thr, half, faults=()):
    """What a kernel with `faults` would return, rounded to the kernel's output types."""
    h = head_ref(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, thr, faults=faults)
    ref = h["ref"]
    return (np.float32(h["loss"]), h["fwd"]["op"].astype(np.float32), h["out"].astype(np.float32),
            ref["dsig"].astype(np.float32), ref["drgb"].astype(np.float16 if half else np.float32))


@pytest.mark.parametrize("half", [False, True])
def test_head_comparator_accepts_the_reference_rounded_to_fp32(half):
    case = _cpu_case(half)
    for w_d in (1e-3, 1e-2, 1.0):
        got = _emulated(*case, 1.0, 2.0 ** 16, w_d, 1e-4, half)
        check_head_dist(got, *case, 1.0, 2.0 ** 16, w_d, 1e-4, half, "fp64 reference")


@pytest.mark.parametrize("fault", ["no_w2d", "sel0", "no_gw", "coef_n", "self_suffix"])
def test_head_comparator_rejects(fault):
    """A dropped w^2 delta / 3, a non-zero selector at k = 0, dL/dw not propagated through the compositing, a
    coefficient off by n_rays, a suffix that includes the sample itself: each is rejected at w_d = 1e-2."""
    half = True
    case = _cpu_case(half)
    got = _emulated(*case, 1.0, 2.0 ** 16, 1e-2, 1e-4, half, faults=(fault,))
    with pytest.raises(AssertionError):
        check_head_dist(got, *case, 1.0, 2.0 ** 16, 1e-2, 1e-4, half, fault)


def test_distortion_entry_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    lib = _lib.load()
    fake = C.c_void_p(0x10000)
    f = lib.ngp_ray_head_fused_distortion
    args = lambda w, ts=fake, dt=F16: (fake, fake, dt, fake, ts, fake, fake, 1.0, 1.0, None, 1e-4, w, fake,  # noqa: E731
                                       None, None, fake, fake, 8, None)
    assert f(*args(-1e-3)) < 0 and b"distortion_w" in lib.ngp_last_error()
    assert f(*args(float("inf"))) < 0 and f(*args(float("nan"))) < 0
    assert f(*args(1e-2, ts=None)) < 0 and b"null" in lib.ngp_last_error()
    assert f(*args(1e-2, dt=7)) < 0 and b"dtype" in lib.ngp_last_error()
    assert f(None, None, F16, None, None, None, None, 1.0, 1.0, None, 1e-4, 1e-2, None, None, None, None, None, 0,
             None) == 0


# ---- GPU: the kernel ---------------------------------------------------------------------------------------------------
def _T(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _N(t):
    return t.detach().cpu().numpy()


def _P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _ST():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def _head(lib, t_in, n, half, loss_scale, thr, w_d, scale_dev=None, plain=False):
    """One launch of ngp_ray_head_fused_distortion (plain: ngp_ray_head_fused) on outputs pre-filled with 9."""
    import torch
    from taichi_nerfs_b200 import _lib
    sig, rgbs, dl, ts, ra, gt = t_in
    S = sig.numel()
    loss_sum, op, rgb = torch.zeros(1, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, 3, device=DEV)
    dsig = torch.full((S,), 9.0, device=DEV)
    drgbs = torch.full((S, 3), 9.0, device=DEV, dtype=torch.float16 if half else torch.float32)
    dt = F16 if half else F32
    if plain:
        _lib.check(lib.ngp_ray_head_fused(_P(sig), _P(rgbs), dt, _P(dl), _P(ra), _P(gt), 1.0, loss_scale,
                                          _P(scale_dev), thr, _P(loss_sum), _P(op), _P(rgb), _P(dsig), _P(drgbs), n,
                                          _ST()))
    else:
        _lib.check(lib.ngp_ray_head_fused_distortion(_P(sig), _P(rgbs), dt, _P(dl), _P(ts), _P(ra), _P(gt), 1.0,
                                                     loss_scale, _P(scale_dev), thr, w_d, _P(loss_sum), _P(op),
                                                     _P(rgb), _P(dsig), _P(drgbs), n, _ST()))
    return loss_sum, op, rgb, dsig, drgbs


def _gpu_case(half, esf, thr):
    """0, 1, 31, 32, 33, 1024 and 5000 samples (alive past 4096: the reverse pass rebuilds the chunk-start carries)
    plus a 4600-sample ray that meets a wall in chunk 131, and short rays sharing their blocks."""
    rng = np.random.default_rng(101 + 2 * half + (esf > 0))
    counts = [0, 1, 31, 32, 33, 1024, 5000, 4600, 12, 300]
    long_x = (0.2e-4, 0.8e-4) if thr > 0.1 else (0.5e-4, 1.5e-4)     # T stays above 0.25 over 5000 samples
    rays_a, sig, deltas, ts = _rays(rng, counts, esf, wall={7: 4200, 9: 100}, long_x=long_x)
    S, n = sig.size, rays_a.shape[0]
    rgbs = (rng.random((S, 3)) * 0.5).astype(np.float16 if half else np.float32)
    gt = rng.random((n, 3)).astype(np.float32)
    return sig, rgbs, deltas, ts, rays_a, gt


@pytest.mark.gpu
@pytest.mark.parametrize("w_d", [1e-3, 1e-2, 1.0])
@pytest.mark.parametrize("esf", [0.0, 1 / 256])
@pytest.mark.parametrize("thr", [1e-4, 0.25])
@pytest.mark.parametrize("half", [False, True])
def test_head_distortion_against_fp64(lib, half, thr, esf, w_d):
    sig, rgbs, deltas, ts, rays_a, gt = case = _gpu_case(half, esf, thr)
    n = rays_a.shape[0]
    scale = 2.0 ** 16
    got = _head(lib, [_T(a) for a in (sig, rgbs, deltas, ts, rays_a, gt)], n, half, scale, thr, w_d)
    got = tuple(_N(t) for t in got)
    h = check_head_dist(got, *case, 1.0, scale, w_d, thr, half, f"half={half} thr={thr} esf={esf} w_d={w_d}")
    r6 = rays_a[6]
    act = h["ref"]["active"]
    assert act[r6[1]:r6[1] + r6[2]].all(), "the 5000-sample ray must stay alive past 4096 samples"
    assert not act[rays_a[7, 1] + 4300], "the 4600-sample ray must stop at its wall"
    assert (h["loss_ray"][rays_a[rays_a[:, 2] > 1, 0]] > 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
def test_head_distortion_device_loss_scale(lib, half):
    """scale_dev holding s == the host constant s, bit for bit (power-of-two scales)."""
    import torch
    sig, rgbs, deltas, ts, rays_a, gt = _gpu_case(half, 0.0, 1e-4)
    t_in = [_T(a) for a in (sig, rgbs, deltas, ts, rays_a, gt)]
    for s in (1.0, 2.0 ** 16, 2.0 ** 19):
        a = _head(lib, t_in, rays_a.shape[0], half, s, 1e-4, 1e-2)
        b = _head(lib, t_in, rays_a.shape[0], half, 12345.0, 1e-4, 1e-2, scale_dev=torch.tensor([s], device=DEV))
        for x, y, name in zip(a[1:], b[1:], ("opacity", "rgb", "dsigma", "drgb")):
            assert torch.equal(x, y), (s, name)
        assert abs(float(a[0]) - float(b[0])) <= 1e-6 * float(a[0])


# ---- GPU: the step -----------------------------------------------------------------------------------------------------
W_D = 1e-2


def _run_step_snap(cfg, w_d, n_steps=1):
    """The graph step of tests/test_gpu_graph_step_grads.py (overlap mode) with the distortion loss; snapshots."""
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from test_gpu_graph_step_grads import N_RAYS, THR, _build, _host_batch, _snapshot
    m, tr, bits = _build(cfg)
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=cfg["spr"], exp_step_factor=cfg["esf"],
                         T_threshold=THR, use_graph=True, overlap_optimizer=True, distortion_loss_w=w_d)
    snaps = []
    for k in range(n_steps):
        o, d, gt, noise = _host_batch(cfg, k)
        fs.step(*(torch.from_numpy(a).cuda() for a in (o, d, gt, noise)))
        snaps.append(_snapshot(fs, m))
    fs.flush()
    del fs, tr, m
    torch.cuda.empty_cache()
    return snaps


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lego_half", "garden_half"])
def test_graph_step_head_stage_with_distortion_against_fp64(name):
    """Stage 4 of tests/test_gpu_graph_step_grads.py with the distortion loss, on the step's own buffers."""
    from test_gpu_graph_step_grads import CONFIGS, THR
    cfg = CONFIGS[name]
    snap = _run_step_snap(cfg, W_D)[0]
    ra = snap["rays_a"]
    assert (ra[:, 2] > 32).any() and snap["counter"][1] == 0
    bg = 1.0 if cfg["esf"] == 0 else 0.0
    got = (snap["loss_sum"][0], snap["opacity"], snap["rgb"], snap["dsig"], snap["drgbs"])
    h = check_head_dist(got, snap["sig"], snap["rgbs"], snap["deltas"], snap["ts"], ra, snap["gt"], bg,
                        snap["scale"], W_D, THR, True, f"{name} step head")
    assert (h["loss_ray"] > 0).any()
    # the distortion's dL/dw is visible at this bound: the same buffers fail the check without it
    with pytest.raises(AssertionError):
        check_head_dist(got, snap["sig"], snap["rgbs"], snap["deltas"], snap["ts"], ra, snap["gt"], bg,
                        snap["scale"], W_D, THR, True, "without dL/dw", faults=("no_gw",))


@pytest.mark.gpu
def test_head_distortion_equals_module_kernel_chain(lib):
    """On a real march (the Lego step's buffers): the fused head == composite_train_fwd -> distortion_fwd / bwd ->
    mse_loss_grad -> composite_train_bwd(dL_dws), each within the fp64 bound of check_head_dist, so within twice it
    of each other; and with w_d = 0 == ngp_ray_head_fused bit for bit."""
    import torch
    from taichi_nerfs_b200 import _lib, ops
    from test_gpu_graph_step_grads import CONFIGS, THR
    snap = _run_step_snap(CONFIGS["lego_half"], W_D)[0]
    sig, rgbs, deltas, ts, ra, gt = (snap[k] for k in ("sig", "rgbs", "deltas", "ts", "rays_a", "gt"))
    n, scale = ra.shape[0], snap["scale"]
    t_in = [_T(a) for a in (sig, rgbs, deltas, ts, ra, gt)]
    fused = tuple(_N(t) for t in _head(lib, t_in, n, True, scale, THR, W_D))
    # the module path's kernels
    t_sig, t_rgbs, t_dl, t_ts, t_ra, t_gt = t_in
    _, op, dep, rgb, ws = ops.composite_train_fwd(t_sig, t_rgbs, t_dl, t_ts, t_ra, THR)
    dist = ops.distortion_fwd(ws, t_dl, t_ts, t_ra)
    dws = ops.distortion_bwd(torch.full((n,), scale * W_D / n, device=DEV), ws, t_dl, t_ts, t_ra)
    ls, g_rgb, g_op = torch.zeros(1, device=DEV), torch.zeros(n, 3, device=DEV), torch.zeros(n, device=DEV)
    _lib.check(lib.ngp_mse_loss_grad(_P(rgb), _P(op), _P(t_gt), 1.0, scale, _P(ls), _P(g_rgb), _P(g_op), n, _ST()))
    dsig, drgbs = ops.composite_train_bwd(g_op, torch.zeros(n, device=DEV), g_rgb, dws, t_sig, t_rgbs, t_dl, t_ts,
                                          t_ra, THR)
    chain = (_N(ls + 3 * W_D * dist.sum()), _N(op), _N(rgb) + (1 - _N(op))[:, None], _N(dsig), _N(drgbs))
    h = check_head_dist(chain, sig, rgbs, deltas, ts, ra, gt, 1.0, scale, W_D, THR, True, "module chain")
    assert np.array_equal(kernel_termination(fused[3], fused[4], ra), kernel_termination(chain[3], chain[4], ra))
    ref = h["ref"]
    tol = 2 * 8 * ref["k"] * U * ref["mag"]
    assert (np.abs(fused[3].astype(np.float64) - chain[3]) <= tol).all(), "dsigma: fused vs chain"
    assert (np.abs(fused[0] - chain[0]) <= 1e-5 * abs(chain[0])), (fused[0], chain[0])
    # w_d = 0: exactly the plain head
    a = _head(lib, t_in, n, True, scale, THR, 0.0)
    b = _head(lib, t_in, n, True, scale, THR, 0.0, plain=True)
    for x, y, name in zip(a[1:], b[1:], ("opacity", "rgb", "dsigma", "drgb")):
        assert torch.equal(x, y), name
    assert abs(float(a[0]) - float(b[0])) <= 1e-6 * float(b[0])


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [False, True])
@pytest.mark.parametrize("use_graph", [False, True])
def test_static_graph_step_with_distortion_equals_autograd_step(lego_bitfield, monkeypatch, use_graph, overlap):
    """StaticTrainStep(distortion_loss_w=1e-2) == NGPTrainer.step(extra_loss=1e-2 * distortion_loss(res).mean()):
    the pattern and criteria of tests/test_gpu_e2e.py::test_static_graph_step_equals_autograd_step."""
    import torch
    from modules.distortion import distortion_loss
    from modules.networks import NGP
    from oracle.train_step import make_rays
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer

    def build():
        torch.manual_seed(3)
        m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
        with torch.no_grad():
            m.pos_encoder.hash_table.mul_(2e3)
            m.density_bitfield.copy_(torch.from_numpy(lego_bitfield))
        return m, NGPTrainer(m, lr=1e-2)

    n = 2048
    o, d = make_rays(n, seed=9)
    o, d = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    gt = torch.rand(n, 3, device='cuda')
    noise = torch.rand(n, device='cuda')

    m1, t1 = build()
    monkeypatch.setattr(torch, 'rand_like', lambda t, **k: noise.clone())
    extra = lambda res: W_D * distortion_loss(res).mean()  # noqa: E731
    losses1 = [float(t1.step(o, d, gt, extra_loss=extra)[0]) for _ in range(3)]
    monkeypatch.undo()

    m2, t2 = build()
    fs = StaticTrainStep(t2, n, samples_per_ray_capacity=64, use_graph=use_graph, overlap_optimizer=overlap,
                         distortion_loss_w=W_D)
    losses2 = [float(fs.step(o, d, gt, noise=noise)) for _ in range(3)]
    fs.flush()
    assert int(fs.counter[0]) > 1000
    for a, b in zip(losses1, losses2):
        assert abs(a - b) < 2e-3 * max(a, 1e-6), (losses1, losses2)
    for p1, p2 in zip(m1.parameters(), m2.parameters()):
        diff = (p1 - p2).abs()
        assert float((diff > 2e-3).float().mean()) < 2e-3, float(diff.max())
    assert t2.step_count == 3 and int(fs.step_dev) == 3
    # The distortion term of the first loss (same parameters, rays and noise) is the module path's.  At w_d = 1e-2 it is
    # ~2e-5 of the loss, inside loss_sum's atomic-order noise, so it is measured at w_d = 10 (~2e-2 of the loss) as the
    # difference of two first-step losses with and without it.
    def first_fused(w):
        _, t = build()
        return float(StaticTrainStep(t, n, samples_per_ray_capacity=64, use_graph=use_graph,
                                     overlap_optimizer=overlap, distortion_loss_w=w).step(o, d, gt, noise=noise))

    def first_module(el):
        _, t = build()
        monkeypatch.setattr(torch, 'rand_like', lambda t, **k: noise.clone())
        loss = float(t.step(o, d, gt, extra_loss=el)[0])
        monkeypatch.undo()
        return loss
    l_f1, l_f0 = first_fused(10.0), first_fused(0.0)
    l_m1, l_m0 = first_module(lambda res: 10.0 * distortion_loss(res).mean()), first_module(None)
    dist_fused, dist_module = l_f1 - l_f0, l_m1 - l_m0
    # Bound.  loss_sum is an fp32 sum of n non-negative per-ray terms in a nondeterministic atomic order: off by at
    # most (n - 1) u of itself, whatever the order; the per-ray MSE terms of the two launches are bit-identical.  The
    # division by 3n and the module path's final additions round by a few u.  5 % covers the difference of the two
    # paths' fp32 distortion sums themselves (measured far below that).
    tol = 0.05 * dist_module + (n + 8) * U * (l_f1 + l_f0 + l_m1 + l_m0)
    assert dist_module > 20 * (n + 8) * U * l_m0, (dist_module, l_m0)   # the term is far above the order noise
    assert abs(dist_fused - dist_module) <= tol, (dist_fused, dist_module, tol)


@pytest.mark.gpu
def test_static_step_rejects_bad_distortion_weight():
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    for w in (-1e-2, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            StaticTrainStep(NGPTrainer(m), 256, samples_per_ray_capacity=8, use_graph=False, distortion_loss_w=w)
    torch.cuda.synchronize()


# ---- GPU: train.py -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_train_graph_step_with_distortion_reaches_psnr(tmp_path, monkeypatch):
    """train.py --graph_step --distortion_loss_w 1e-2 on the analytic scene (the configuration of
    tests/test_gpu_e2e.py::test_training_on_analytic_scene_reaches_psnr)."""
    import train
    from test_gpu_e2e import _small_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _small_dataset})
    psnrs = train.main(['--dataset_name', 'synthetic', '--half_opt', '--batch_size', '4096', '--max_steps', '400',
                        '--graph_step', '--distortion_loss_w', '1e-2'])
    assert min(psnrs) > 22.0, psnrs


@pytest.mark.gpu
def test_train_graph_step_still_refuses_the_deployment_model(tmp_path, monkeypatch):
    import train
    from test_gpu_e2e import _small_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _small_dataset})
    with pytest.raises(ValueError, match="stock NGP architecture"):
        train.main(['--dataset_name', 'synthetic', '--batch_size', '1024', '--max_steps', '1', '--graph_step',
                    '--deployment', '--distortion_loss_w', '1e-2'])
