"""The kernels of the graph-captured training step (taichi_nerfs_b200/fast_step.py) and of the optimizer update that
both training paths share, one kernel at a time on fixed inputs, against a plain high-precision reference.

- Hash forward with the AABB folded in and the row count read on the device: bit-exact against the oracle.
- Hash backward by level group: an fp64 scatter with a bound that holds for any atomic order.
- GradScaler's inf check raised at the source by the MLP and hash backward kernels ("inf at source"): the flag is
  raised exactly when the gradient buffer holds a non-finite value.  Not covered: an fp32 overflow inside the atomic
  sum itself.  Every contribution is bounded by the fp16 dL/demb (65504), so that would take ~1e34 contributions to
  one entry.
- The optimizer bookkeeping (step reset, LR schedule and bias corrections, Adam, GradScaler update) over a scripted
  trajectory against torch's CosineAnnealingLR, torch._amp_update_scale_ and an fp64 torch.optim.Adam.
- The fp16 gradient transport of the multi-rank update.
- The per-ray head on rays long enough to take the transmittance-recompute path, against fp64 compositing.
- Argument validation of these entry points (CPU only).

Every device-count (n_dev) test allocates n_max + PAD rows, pre-fills outputs and pad with a sentinel and passes
n_max: a kernel that ignored the clamp would write sentinel rows, never outside its buffers.
"""
import ctypes as C
import functools
import math
import warnings

import numpy as np
import pytest
import torch

from taichi_nerfs_b200.layout import make_hash_layout

from composite_ref import _check_composite_bwd, np_composite_f64
from hash_ref import (PAD, _aabb6, _check_scatter, _level_ranges, _level_slice, _normalise, _ray_points,
                      _world_points, n_dev_cases, np_hash_bwd_f64, rows_of)

DEV = "cuda"
U = 2.0 ** -24          # fp32 unit roundoff
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


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def i32(v):
    return torch.tensor([v], device=DEV, dtype=torch.int32)


# ---- hash grid helpers --------------------------------------------------------------------------------------------
SCENES = {"lego": (0.5, 1024), "garden": (16.0, 4096)}   # scale of the box, finest resolution


@functools.lru_cache(maxsize=None)
def _layout(max_res):
    return make_hash_layout(2 ** 19, 16, 16, max_res, 2)


@functools.lru_cache(maxsize=4)
def _table(max_res, half):
    rng = np.random.default_rng(max_res + half)
    t = rng.standard_normal(_layout(max_res).total_param_size).astype(np.float32)
    return (t * 0.1).astype(np.float16) if half else t


# ---- 1. hash forward, _dyn with the AABB folded in ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_max", [1, 511, 512, 513])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("scene", list(SCENES))
def test_hash_fwd_dyn_aabb_bit_exact(lib, oracle, scene, half, n_max):
    """ngp_hash_encode_fwd_dyn with aabb6 and n_dev == the oracle on the fp32-normalised points, bit for bit, on the
    rows [0, min(n_max, max(n_dev, 0))); every other row keeps the sentinel."""
    scale, max_res = SCENES[scene]
    lay = _layout(max_res)
    cl = lay.as_ctypes()
    table = _table(max_res, half)
    rng = np.random.default_rng(1000 * n_max + max_res + half)
    x = _world_points(rng, n_max + PAD, scale)
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


# ---- 2. hash backward by level group against an fp64 scatter --------------------------------------------------------
def _bwd_inputs(rng, n, half):
    xn = _ray_points(rng, n)
    dout = rng.standard_normal((n, 32)).astype(np.float32)
    dout[rng.random(n) < 0.1] = 0.0                            # skipped rows
    lv = rng.random((n, 16)) < 0.05                            # single levels with dy = (0, 0)
    dout.reshape(n, 16, 2)[lv] = 0.0
    dout.reshape(n, 16, 2)[rng.random((n, 16)) < 0.05, 1] = 0.0   # dy = (x, 0) still contributes
    return xn, (dout.astype(np.float16) if half else dout)


@pytest.mark.gpu
@pytest.mark.parametrize("group", ["all", "dense", "hashed_coarse", "hashed_fine", "last", "level3", "inner"])
@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_levels_fp64_bound(lib, half, group):
    lay = _layout(1024)
    cl = lay.as_ctypes()
    a, b = _level_ranges(lay)[group]
    rng = np.random.default_rng(7 + half)
    n = 20000
    xn, dout = _bwd_inputs(rng, n, half)
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    g, t_x, t_d = T(prefill), T(xn), T(dout)   # (named: a temporary's memory could be reused before the launch)
    chk(lib.ngp_hash_encode_bwd_levels(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n, None, None,
                                       a, b, None, ST()))
    ref, mag, cnt = np_hash_bwd_f64(xn, dout, lay, half, range(a, b))
    lo, hi = _level_slice(lay, a, b)
    assert cnt[lo:hi].max() > 1   # the run accumulation is exercised
    _check_scatter(N(g), prefill, ref, mag, cnt, lo, hi, f"levels [{a},{b})")


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
def test_hash_bwd_levels_dyn_aabb(lib, half):
    """World positions normalised inside the kernel and the row count read on the device: rows at or beyond
    min(n_max, n_dev) contribute nothing."""
    scale = 0.5
    lay = _layout(1024)
    cl = lay.as_ctypes()
    rng = np.random.default_rng(11 + half)
    n_max = 3000
    xn, dout = _bwd_inputs(rng, n_max + PAD, half)
    xw = (xn * np.float32(2 * scale) - np.float32(scale)).astype(np.float32)
    xw[: n_max // 7] = _world_points(rng, n_max // 7, scale)       # face points too
    xnn = _normalise(xw, scale)
    prefill = (rng.standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    t_x, t_d = T(xw), T(dout)
    for nd in n_dev_cases(n_max):
        g = T(prefill)
        chk(lib.ngp_hash_encode_bwd_levels(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n_max,
                                           P(i32(nd)), _aabb6(scale), 0, lay.levels, None, ST()))
        m = rows_of(nd, n_max)
        ref, mag, cnt = np_hash_bwd_f64(xnn[:m], dout[:m], lay, half, range(lay.levels))
        _check_scatter(N(g), prefill, ref, mag, cnt, 0, lay.total_param_size, f"n_dev={nd}")


# ---- 3. inf at source -------------------------------------------------------------------------------------------------
def _mlp_weights_np(rng):
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    return [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]


class _Net:
    """Inputs of one MLP + hash backward as the graph step holds them: n_max + PAD rows, n_dev on the device."""

    def __init__(self, seed, n_max, random_xyz=False):
        from taichi_nerfs_b200 import ops
        rng = np.random.default_rng(seed)
        R = n_max + PAD
        self.n_max, self.lay = n_max, _layout(1024)
        self.cl = self.lay.as_ctypes()
        self.P = self.lay.total_param_size
        self.emb = T(rng.standard_normal((R, 32)).astype(np.float16))
        self.dirs = T(rng.standard_normal((R, 3)).astype(np.float32))
        self.ws = [T(w) for w in _mlp_weights_np(rng)]
        self.wst, self._keep = ops._mlp_weights(self.ws)
        self.xyz = rng.random((R, 3), dtype=np.float32) if random_xyz else _ray_points(rng, R)
        self.dsig = (rng.standard_normal(R) * 1e-2).astype(np.float32)
        self.drgb = (rng.standard_normal((R, 3)) * 1e-2).astype(np.float16)

    def mlp_bwd(self, lib, n_dev, dsig, drgb, grad_w, demb, found):
        # padded like every other buffer: the h block of a kernel that ignored the clamp would run into the rgb block
        # (at n_max * 16 halves), never past the allocation
        save = torch.zeros(int(lib.ngp_mlp_save_bytes(self.n_max + PAD)), device=DEV, dtype=torch.uint8)
        sig = torch.zeros(self.n_max + PAD, device=DEV)
        rgb = torch.zeros(self.n_max + PAD, 3, device=DEV, dtype=torch.float16)
        chk(lib.ngp_mlp_fwd_dyn(P(self.emb), F16, P(self.dirs), C.byref(self.wst), P(sig), P(rgb), P(save),
                                self.n_max, P(n_dev), ST()))
        chk(lib.ngp_mlp_bwd_dyn(P(self.emb), F16, P(self.dirs), C.byref(self.wst), P(save), P(dsig), P(drgb),
                                P(demb), P(grad_w), self.n_max, P(n_dev), P(found), ST()))


def _check_finite(lib, t):
    f = torch.zeros(1, device=DEV, dtype=torch.int32)
    chk(lib.ngp_check_finite(P(t), t.numel(), P(f), ST()))
    return int(f)


INF_CASES = (["clean"]
             + [f"{tgt}_{v}_{where}" for where in ("in", "beyond", "pad") for tgt in ("dsig", "drgb")
                for v in ("nan", "+inf", "-inf")]
             + ["demb_inf_other_level", "zero_dy_nan_xyz"])


@pytest.mark.gpu
@pytest.mark.parametrize("case", INF_CASES)
def test_inf_at_source_flag_equals_check_finite(lib, case):
    """MLP backward then hash backward on the same buffers with one found_inf, as the graph step enqueues them:
    flag raised <=> the flat gradient holds a non-finite value, and poison outside the processed rows or levels
    raises nothing.  The flag is checked after each launch, so that each kernel must raise it for its own slice:
    a poisoned dsig / drgb row also poisons dL/demb, and the hash backward alone would raise it too."""
    net = _Net(21, 4000)
    n_dev = 3000
    vals = {"nan": np.nan, "+inf": np.inf, "-inf": -np.inf}
    dsig, drgb, xyz = net.dsig.copy(), net.drgb.copy(), net.xyz.copy()
    levels = (0, 16)
    expect = None
    if case != "clean" and case.split("_")[0] in ("dsig", "drgb"):
        tgt, v, where = case.split("_")
        row = {"in": 1234, "beyond": 3500, "pad": 4000 + 17}[where]
        if tgt == "dsig":
            dsig[row] = vals[v]
        else:
            drgb[row, 1] = vals[v]
        expect = where == "in"
    elif case == "zero_dy_nan_xyz":
        dsig[777], drgb[777] = 0.0, 0.0
        xyz[777] = np.nan
        expect = False
    elif case == "demb_inf_other_level":
        levels = (0, 8)
    flat = torch.zeros(net.P + 9408, device=DEV)
    demb = torch.zeros(net.n_max + PAD, 32, device=DEV, dtype=torch.float16)
    found = torch.zeros(1, device=DEV, dtype=torch.int32)
    nd = i32(n_dev)
    net.mlp_bwd(lib, nd, T(dsig), T(drgb), flat[net.P:], demb, found)
    flag_mlp, bad_mlp = int(found), _check_finite(lib, flat[net.P:])
    assert flag_mlp == bad_mlp, f"{case}: MLP backward found_inf={flag_mlp}, its weight gradient non-finite={bad_mlp}"
    if expect is not None:
        assert flag_mlp == int(expect), f"{case}: MLP backward"
    if case == "demb_inf_other_level":
        demb[100, 2 * 12] = float("inf")
        expect = False
    t_xyz = T(xyz)
    chk(lib.ngp_hash_encode_bwd_levels(P(t_xyz), P(demb), F16, C.byref(net.cl), P(flat), net.n_max, P(nd), None,
                                       levels[0], levels[1], P(found), ST()))
    flag, bad = int(found), _check_finite(lib, flat)
    assert flag == bad, f"{case}: found_inf={flag} but the gradient {'is' if bad else 'is not'} non-finite"
    if expect is not None:
        assert flag == int(expect), case


@pytest.mark.gpu
@pytest.mark.parametrize("level", [0, 9, 15])
def test_hash_bwd_flags_an_early_flush(lib, level):
    """A non-finite dL/demb at the first sample of a lane's 16-sample chunk, at one level only: on fine levels every
    sample of random positions opens a new cell, so the poisoned run is flushed long before the lane's last flush."""
    net = _Net(22, 4096, random_xyz=True)
    demb = (torch.randn(net.n_max + PAD, 32, device=DEV) * 1e-2).half()
    flat = torch.zeros(net.P, device=DEV)
    found = torch.zeros(1, device=DEV, dtype=torch.int32)
    demb[512 * 3 + 16 * 5, 2 * level + 1] = float("nan")
    t_xyz = T(net.xyz)
    chk(lib.ngp_hash_encode_bwd_levels(P(t_xyz), P(demb), F16, C.byref(net.cl), P(flat), net.n_max, None, None,
                                       0, 16, P(found), ST()))
    assert _check_finite(lib, flat) == 1
    assert int(found) == 1


@pytest.mark.gpu
def test_mlp_bwd_dyn_equals_mlp_bwd_on_first_rows(lib):
    """ngp_mlp_bwd_dyn on n_max rows with n_dev == ngp_mlp_bwd on the first n rows: dL/demb bit-identical, weight
    gradients within 2e-5 of their maximum (fp32 atomics); demb rows >= n keep the sentinel; n = 0 adds nothing."""
    from taichi_nerfs_b200 import ops
    net = _Net(23, 5000)
    rng = np.random.default_rng(24)
    prefill = (rng.uniform(-1, 1, 9408) * 1e-3).astype(np.float32)
    dsig, drgb = T(net.dsig), T(net.drgb)
    for nd in n_dev_cases(net.n_max):
        n = rows_of(nd, net.n_max)
        gw = T(prefill)
        demb = torch.full((net.n_max + PAD, 32), -7.0, device=DEV, dtype=torch.float16)
        net.mlp_bwd(lib, i32(nd), dsig, drgb, gw, demb, None)
        got_w = N(gw)
        if n == 0:
            assert np.array_equal(got_w.view(np.uint32), prefill.view(np.uint32)), f"n_dev={nd}: grad_w touched"
        else:
            de_ref, gw_ref = ops.mlp_bwd(net.emb[:n], net.dirs[:n], net.ws, dsig[:n], drgb[:n])
            assert torch.equal(demb[:n], de_ref), f"n_dev={nd}: dL/demb differs"
            gw_ref = N(gw_ref).astype(np.float64)
            err = np.abs(got_w.astype(np.float64) - prefill - gw_ref).max()
            assert err <= 2e-5 * np.abs(gw_ref).max() + 4 * U, f"n_dev={nd}: grad_w err {err}"
        assert bool((demb[n:] == -7.0).all()), f"n_dev={nd}: demb row >= n written"


# ---- 4. optimizer bookkeeping against torch ---------------------------------------------------------------------------
LR0 = float(np.float32(1e-2))           # the kernel receives fp32 constants
LR_MIN = float(np.float32(1e-2 / 30))
B1, B2, EPS = float(np.float32(0.9)), float(np.float32(0.999)), 1e-15
MAX_STEPS, INTERVAL, ITERS = 25, 3, 40

# (initial scale, iterations whose gradient holds an inf/NaN)
SCRIPTS = {
    # clean steps; a skip right after the growth at iteration 2; back-to-back skips; steps past max_steps
    "mixed": (2.0 ** 16, {3, 9, 10, 11, 17, 24, 31}),
    "first_skip": (2.0 ** 16, {0, 1, 6}),
    # grows to 2^126 and 2^127, then must not grow to inf
    "huge_scale": (2.0 ** 125, {20}),
}


def _cosine_scheduler():
    dummy = torch.nn.Parameter(torch.zeros(1, dtype=torch.float64))
    opt = torch.optim.SGD([dummy], lr=LR0)
    return opt, torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=MAX_STEPS, eta_min=LR_MIN)


def test_cosine_scheduler_is_the_closed_form():
    """CPU: torch's recursive CosineAnnealingLR agrees with the closed form the kernel evaluates, over the whole
    schedule, to ~1e-15: the GPU trajectory test can compare against either."""
    opt, sched = _cosine_scheduler()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for s in range(MAX_STEPS + 1):
            closed = LR_MIN + (LR0 - LR_MIN) * (1 + math.cos(math.pi * s / MAX_STEPS)) / 2
            assert abs(sched.get_last_lr()[0] - closed) <= 1e-15, s
            opt.step()
            sched.step()


def _within_ulp(got, want64, what):
    want = np.float32(want64)
    assert abs(float(got) - float(want)) <= float(np.spacing(np.abs(want))), f"{what}: {got!r} vs {want!r}"


def _adam_case(n, variant, script):
    return pytest.param(n, variant, script, id=f"{n}-{variant}-{script}")


# variant: (fp16 shadow, zero_grad, element offset of a 16-byte aligned sub-slice view, world size, clear_found_inf)
VARIANTS = {"full": (True, 1, 0, 1, 1), "view": (True, 1, 4, 2, 0), "bare": (False, 0, 4, 1, 0)}
ADAM_SIZES = [1, 3, 4, 5, 1023, 11420064 // 8 + 3]
ADAM_CASES = ([_adam_case(n, v, "mixed") for n in ADAM_SIZES for v in VARIANTS]
              + [_adam_case(n, v, "first_skip") for n in (5, 1023) for v in ("full", "view")]
              + [_adam_case(n, "full", "huge_scale") for n in (5, 1023)])


@pytest.mark.gpu
@pytest.mark.parametrize("n,variant,script", ADAM_CASES)
def test_optimizer_trajectory_against_torch(lib, oracle, n, variant, script):
    """ngp_step_reset -> [backward: gradient + found_inf] -> ngp_adam_hyper_update -> ngp_adam_step_dyn ->
    ngp_loss_scale_update, as NGPTrainer.enqueue_update enqueues them, for ITERS iterations."""
    shadow_on, zero_grad, off, world, clear = VARIANTS[variant]
    scale, skips = SCRIPTS[script]
    rng = np.random.default_rng(n + 31 * off)
    p0 = rng.standard_normal(n).astype(np.float32)
    R = n + 2 * off

    def buf(init, dtype=torch.float32):
        b = torch.full((R,), -3.0, device=DEV, dtype=dtype)   # guards around the view
        b[off:off + n] = init
        return b

    b_p, b_g, b_m, b_v = buf(T(p0)), buf(0.0), buf(0.0), buf(0.0)
    b_sh = buf(T(p0).half(), torch.float16) if shadow_on else None
    p, g, m, v = (b[off:off + n] for b in (b_p, b_g, b_m, b_v))
    sh = None if b_sh is None else b_sh[off:off + n]
    step_dev, found = i32(0), i32(0)
    counter2, loss_sum, batch = torch.tensor([5, 6], device=DEV, dtype=torch.int32), torch.ones(1, device=DEV), i32(0)
    hyper = torch.zeros(4, device=DEV)
    hyper[2] = float(np.float32(1) / (np.float32(scale) * np.float32(world)))
    state = torch.tensor([scale, 0.0], device=DEV)

    # references: torch's scheduler, GradScaler update and fp64 Adam
    sopt, sched = _cosine_scheduler()
    ref_scale, ref_tracker = torch.tensor([scale], dtype=torch.float32), torch.zeros(1, dtype=torch.int32)
    p64 = torch.nn.Parameter(torch.from_numpy(p0.astype(np.float64)))
    adam64 = torch.optim.Adam([p64], lr=LR0, betas=(B1, B2), eps=EPS)
    pmax = np.abs(p0).astype(np.float64)
    t, prev_grew, grew_then_skipped = 0, False, False
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for it in range(ITERS):
            skip = it in skips
            # the scheduler steps every iteration, skipped or not (train.py:201); the kernel holds lr_min past
            # max_steps, where torch's schedule would rise again
            lr_s = sched.get_last_lr()[0] if it <= MAX_STEPS else LR_MIN
            if it < MAX_STEPS:
                sopt.step()
                sched.step()
            cur_scale = float(ref_scale)
            g_true = (rng.standard_normal(n) * 1e-3).astype(np.float32)
            g_buf = (g_true * np.float32(cur_scale) * np.float32(world)).astype(np.float32)   # exact: powers of two
            if skip:
                g_buf[rng.integers(0, n)] = np.nan
            chk(lib.ngp_step_reset(P(counter2), P(loss_sum), P(found), P(batch), ST()))
            g.copy_(T(g_buf))
            found.fill_(int(skip))
            before = [N(x).copy() for x in (p, m, v)] + ([N(sh).copy()] if sh is not None else [])
            inv_prev = float(hyper[2])
            chk(lib.ngp_adam_hyper_update(P(step_dev), LR0, LR_MIN, MAX_STEPS, B1, B2, -1.0, P(found), P(hyper),
                                          ST()))
            chk(lib.ngp_adam_step_dyn(P(p), P(g), P(m), P(v), P(sh), P(found), P(hyper), B1, B2, EPS, zero_grad, n,
                                      ST()))
            chk(lib.ngp_loss_scale_update(P(state), P(found), 2.0, 0.5, INTERVAL, float(world), P(hyper), clear, ST()))
            after = [N(x) for x in (p, m, v)] + ([N(sh)] if sh is not None else [])
            hy = N(hyper)

            # bookkeeping
            assert int(step_dev) == it + 1
            assert int(batch) == it + 1 and int(counter2.abs().sum()) == 0 and float(loss_sum) == 0.0
            if not skip:
                t += 1
            assert int(hy.view(np.int32)[3]) == t, f"iteration {it}: Adam's step count"
            te = max(t, 1)   # a skipped first step still evaluates the bias corrections at t = 1
            _within_ulp(hy[0], lr_s / (1 - B1 ** te), f"iteration {it}: lr / (1 - beta1^t)")
            _within_ulp(hy[1], math.sqrt(1 - B2 ** te), f"iteration {it}: sqrt(1 - beta2^t)")
            torch._amp_update_scale_(ref_scale, ref_tracker, torch.tensor([float(skip)]), 2.0, 0.5, INTERVAL)
            grew_then_skipped |= skip and prev_grew
            prev_grew = float(ref_scale) > cur_scale
            st_ = N(state)
            assert st_[0] == float(ref_scale) and int(st_.view(np.int32)[1]) == int(ref_tracker), \
                f"iteration {it}: scale state {st_[0]}, {st_.view(np.int32)[1]} vs torch {float(ref_scale)}, " \
                f"{int(ref_tracker)}"
            with np.errstate(over="ignore"):
                want_inv = np.float32(1) / (np.float32(st_[0]) * np.float32(world))
            assert hy[2] == want_inv, f"iteration {it}: hyper[2] {hy[2]} vs 1/(scale*world) {want_inv}"
            assert int(found) == (0 if clear else int(skip)), f"iteration {it}: found_inf after the update"
            gg = N(g)
            if zero_grad:
                assert not gg.any(), f"iteration {it}: gradient not zeroed"
            else:
                assert np.array_equal(gg.view(np.uint32), g_buf.view(np.uint32))

            if skip:
                for b, a, name in zip(before, after, ("param", "exp_avg", "exp_avg_sq", "shadow")):
                    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"iteration {it}: {name} changed"
                continue
            # fp32 oracle from the same state, with the host-side lr, t and inv_scale
            op_, om_, ov_ = before[0].copy(), before[1].copy(), before[2].copy()
            oracle.adam_step(op_, g_buf.copy(), om_, ov_, lr_s, t, beta1=B1, beta2=B2, eps=EPS, inv_scale=inv_prev)
            np.testing.assert_allclose(after[0], op_, rtol=2e-6, atol=1e-7, err_msg=f"iteration {it}: param")
            # m + (g - m)(1 - beta1) cancels where g ~ m: its rounding is relative to |m| + |g|, not to the result
            gg = np.abs(g_buf.astype(np.float64) * inv_prev)
            m_err = np.abs(after[1].astype(np.float64) - om_)
            assert (m_err <= 2e-6 * np.abs(om_) + 4 * U * (np.abs(before[1]) + gg)).all(), f"iteration {it}: exp_avg"
            np.testing.assert_allclose(after[2], ov_, rtol=2e-6, atol=1e-18, err_msg=f"iteration {it}: exp_avg_sq")
            if sh is not None:
                assert np.array_equal(after[3].view(np.uint16), after[0].astype(np.float16).view(np.uint16))
            # fp64 Adam on the unscaled gradient
            for grp in adam64.param_groups:
                grp["lr"] = lr_s
            p64.grad = torch.from_numpy(g_buf.astype(np.float64) * inv_prev)
            adam64.step()
            pmax = np.maximum(pmax, np.abs(p64.detach().numpy()))
    if script == "mixed":
        assert grew_then_skipped, "the script must skip right after a growth"
    got = N(p).astype(np.float64)
    tol = t * (np.spacing(pmax.astype(np.float32)).astype(np.float64) + LR0 * 2.0 ** -20)
    err = np.abs(got - p64.detach().numpy())
    assert (err <= tol).all(), f"fp64 Adam: max err/tol {(err / tol).max():.3f}"
    for b in [b_p, b_g, b_m, b_v] + ([b_sh] if b_sh is not None else []):
        guards = torch.cat([b[:off], b[off + n:]])
        assert bool((guards == -3.0).all()), "wrote outside the view"


@pytest.mark.gpu
def test_step_reset_every_pointer_optional(lib):
    c2 = torch.tensor([5, 6], device=DEV, dtype=torch.int32)
    ls, fi, bc = torch.tensor([3.5], device=DEV), i32(1), i32(41)
    chk(lib.ngp_step_reset(None, None, None, None, ST()))
    torch.cuda.synchronize()
    assert N(c2).tolist() == [5, 6] and float(ls) == 3.5 and int(fi) == 1 and int(bc) == 41
    chk(lib.ngp_step_reset(P(c2), None, None, None, ST()))
    assert N(c2).tolist() == [0, 0] and float(ls) == 3.5 and int(fi) == 1 and int(bc) == 41
    chk(lib.ngp_step_reset(None, P(ls), None, None, ST()))
    assert float(ls) == 0.0 and int(fi) == 1 and int(bc) == 41
    chk(lib.ngp_step_reset(None, None, P(fi), None, ST()))
    assert int(fi) == 0 and int(bc) == 41
    for k in range(3):
        chk(lib.ngp_step_reset(None, None, None, P(bc), ST()))
        assert int(bc) == 42 + k


@pytest.mark.gpu
def test_lr_stays_at_lr_min_past_max_steps(lib):
    step_dev, hyper = i32(MAX_STEPS - 1), torch.zeros(4, device=DEV)
    hyper.view(torch.int32)[3] = 99
    for s in range(MAX_STEPS - 1, MAX_STEPS + 6):
        chk(lib.ngp_adam_hyper_update(P(step_dev), LR0, LR_MIN, MAX_STEPS, B1, B2, 0.25, None, P(hyper), ST()))
        hy = N(hyper)
        t = int(hy.view(np.int32)[3])
        assert t == 100 + s - (MAX_STEPS - 1) and hy[2] == 0.25
        want = (LR_MIN + (LR0 - LR_MIN) * (1 + math.cos(math.pi * s / MAX_STEPS)) / 2) if s <= MAX_STEPS else LR_MIN
        _within_ulp(hy[0], want / (1 - B1 ** t), f"s={s}")


# ---- 5. fp16 gradient transport -------------------------------------------------------------------------------------
def _pack_values(rng, n):
    special = np.array([0.0, -0.0, 65504.0, -65504.0, 65519.99, 65520.0, -65520.0, 1e5, np.inf, -np.inf,
                        2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, -1.5 * 2.0 ** -24, 2.0 ** -14, 2.0 ** -14 * (1 - 2 ** -11),
                        1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 2049.0, 2051.0, 1e-9, -1e-9, 7e-6],
                       np.float32)
    x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 5, n)).astype(np.float32)
    pos = rng.permutation(n)[: min(n, len(special))]
    x[pos] = special[: pos.size]
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("n", list(range(1, 18)) + [100003])
def test_grad_pack_f16_rounds_like_torch_half(lib, n):
    rng = np.random.default_rng(n)
    x = _pack_values(rng, n)
    if n >= 6:
        x[n // 2] = np.nan
    want = torch.from_numpy(x).half().numpy()
    out = torch.full((n + 8,), 123.0, device=DEV, dtype=torch.float16)
    t_x = T(x)
    chk(lib.ngp_grad_pack_f16(P(t_x), P(out), n, ST()))
    got = N(out)
    nan = np.isnan(x)
    assert np.isnan(got[:n][nan]).all()
    assert np.array_equal(got[:n][~nan].view(np.uint16), want[~nan].view(np.uint16)), \
        f"differs at {np.flatnonzero(got[:n][~nan].view(np.uint16) != want[~nan].view(np.uint16))[:5]}"
    assert (got[n:] == 123.0).all()


def _finite_values(rng, n, half):
    if half:
        extremes = np.array([65504.0, -65504.0, 2.0 ** -24, -(2.0 ** -24), -0.0, 2.0 ** -14 * 0.5], np.float16)
        x = (rng.standard_normal(n) * 100).astype(np.float16)
    else:
        extremes = np.array([3.4028235e38, -3.4028235e38, 1e-45, -1e-45, -0.0, 1e-40], np.float32)
        x = (rng.standard_normal(n) * 1e30).astype(np.float32)
    x[rng.permutation(n)[: min(n, extremes.size)]] = extremes[: min(n, extremes.size)]
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("half", [True, False], ids=["f16", "f32"])
def test_check_finite_every_head_and_tail_position(lib, half):
    """One non-finite value at the first element, at the last element of the vectorised part and at every tail
    element, for n = 1..17 and a large n; clean buffers of extreme finite values never raise the flag, and the flag
    is only ever raised, never cleared."""
    fn = lib.ngp_check_finite_f16 if half else lib.ngp_check_finite
    vec, dt = (8, np.float16) if half else (4, np.float32)
    rng = np.random.default_rng(5 + half)
    for n in list(range(1, 18)) + [100003]:
        nv = n // vec * vec
        positions = sorted({0, max(nv - 1, 0)} | set(range(nv, n)))
        bads = [np.inf, -np.inf, np.nan]
        stride = (n + 7) // 8 * 8
        clean = _finite_values(rng, n, half)
        cases = [(pos, b) for pos in positions for b in bads]
        host = np.zeros((len(cases) + 2, stride), dt)
        host[:, :n] = clean
        for k, (pos, b) in enumerate(cases):
            host[k, pos] = b
        host[len(cases) + 1, 0] = np.nan                # raised flag, poisoned buffer
        buf = T(host)
        flags = torch.zeros(len(cases) + 2, device=DEV, dtype=torch.int32)
        flags[len(cases):] = 1                           # pre-raised: a clean buffer must not clear it
        es = buf.element_size()
        for k in range(len(cases) + 2):
            chk(fn(C.c_void_p(buf.data_ptr() + k * stride * es), n, C.c_void_p(flags.data_ptr() + 4 * k), ST()))
        fl = N(flags)
        missed = [cases[k] for k in range(len(cases)) if fl[k] != 1]
        assert not missed, f"n={n}: non-finite value missed at (position, value) {missed[:4]}"
        assert fl[len(cases)] == 1 and fl[len(cases) + 1] == 1, f"n={n}: flag cleared"
        clean_flag = torch.zeros(1, device=DEV, dtype=torch.int32)
        chk(fn(C.c_void_p(buf.data_ptr() + len(cases) * stride * es), n, P(clean_flag), ST()))
        assert int(clean_flag) == 0, f"n={n}: flag raised by finite values"


def _adam_state(rng, n):
    p = rng.standard_normal(n).astype(np.float32)
    m = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    v = (rng.random(n) * 1e-6).astype(np.float32)
    return p, m, v


def _hyper(t, inv_scale):
    h = torch.tensor([LR0 / (1 - B1 ** t), math.sqrt(1 - B2 ** t), inv_scale, 0.0], device=DEV)
    h.view(torch.int32)[3] = t
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("with_f32_buffer", [True, False])
@pytest.mark.parametrize("n", ADAM_SIZES)
def test_adam_g16_bit_identical_to_adam_on_float(lib, n, with_f32_buffer):
    """Adam reading the fp16 transport buffer == Adam reading the same values as fp32 (only the load differs); the
    fp32 accumulation buffer is zeroed, skipped or not, and may be absent."""
    rng = np.random.default_rng(n)
    p, m, v = _adam_state(rng, n)
    g16 = T((rng.standard_normal(n) * 2000).astype(np.float16))
    g16[: min(n, 2)] = torch.tensor([2.0 ** -24, -65504.0][: min(n, 2)], dtype=torch.float16)
    hyper = _hyper(7, 2.0 ** -16)
    for skip in (0, 1):
        found = i32(skip)
        pa, ma, va, sa = T(p), T(m), T(v), torch.zeros(n, device=DEV, dtype=torch.float16)
        pb, mb, vb, sb = T(p), T(m), T(v), torch.zeros(n, device=DEV, dtype=torch.float16)
        gf = g16.float()
        chk(lib.ngp_adam_step_dyn(P(pa), P(gf), P(ma), P(va), P(sa), P(found), P(hyper), B1, B2, EPS, 1, n, ST()))
        buf = torch.full((n,), 5.0, device=DEV) if with_f32_buffer else None
        chk(lib.ngp_adam_step_dyn_g16(P(pb), P(g16), P(buf), P(mb), P(vb), P(sb), P(found), P(hyper), B1, B2, EPS, n,
                                      ST()))
        for a, b, name in ((pa, pb, "param"), (ma, mb, "exp_avg"), (va, vb, "exp_avg_sq"), (sa, sb, "shadow")):
            assert torch.equal(a.view(torch.int16 if a.dtype == torch.float16 else torch.int32),
                               b.view(torch.int16 if b.dtype == torch.float16 else torch.int32)), f"skip={skip}: {name}"
        if skip:
            assert np.array_equal(N(pb), p)
        else:
            assert not np.array_equal(N(pb), p)
        if buf is not None:
            assert not bool(buf.any()), f"skip={skip}: fp32 buffer not zeroed"


# ---- 6. compositing: long rays and the device loss scale -------------------------------------------------------------
def _long_rays(rng, half):
    """Rays for the c >= kChunkCap (128 chunks of 32 = 4096 samples) path that recomputes the chunk-start
    transmittance: one of 5000 samples that stays above the threshold, one that terminates in chunk 131 on a dense
    wall, plus short and empty rays sharing their blocks."""
    counts = [5000, 4600, 37, 0, 300, 1]
    sd = []
    for k, c in enumerate(counts):
        x = rng.uniform(0.5e-3, 1.5e-3, c)
        if k == 1:
            x[4200] = 30.0
        if k == 4:
            x[:] = rng.uniform(0.005, 0.02, c)
            x[100] = 40.0
        sd.append(x)
    sd = np.concatenate(sd)
    S = sd.size
    deltas = rng.uniform(1e-3, 3e-3, S).astype(np.float32)
    sig = (sd / deltas).astype(np.float32)
    rgbs = (rng.random((S, 3)) * 0.5).astype(np.float16 if half else np.float32)
    ts = np.cumsum(deltas).astype(np.float32)
    counts = np.array(counts)
    n = counts.size
    rays_a = np.stack([rng.permutation(n), np.cumsum(counts) - counts, counts], 1).astype(np.int32)
    return rays_a, sig, rgbs, deltas, ts


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
def test_composite_train_bwd_long_rays_fp64(lib, half):
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(61 + half)
    rays_a, sig, rgbs, deltas, ts = _long_rays(rng, half)
    n, S = rays_a.shape[0], sig.size
    go, gd = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    gr, gw = rng.standard_normal((n, 3)).astype(np.float32), rng.standard_normal(S).astype(np.float32)
    ref = np_composite_f64(sig, rgbs, deltas, ts, rays_a, 1e-4, go, gd, gr, gw)
    assert ref["active"][rays_a[0, 1]:rays_a[0, 1] + 5000].all() and ref["active"].sum() < S
    dsig, drgbs = ops.composite_train_bwd(T(go), T(gd), T(gr), T(gw), T(sig), T(rgbs), T(deltas), T(ts), T(rays_a),
                                          1e-4)
    _check_composite_bwd(N(dsig), N(drgbs), ref, half, "composite_train_bwd")


def _head_ref(rays_a, sig, rgbs, deltas, ts, gt, bg, scale):
    n, S = rays_a.shape[0], sig.size
    z = np.zeros(n)
    fwd = np_composite_f64(sig, rgbs, deltas, ts, rays_a, 1e-4, z, z, np.zeros((n, 3)), np.zeros(S))
    out = fwd["rgb"] + bg * (1 - fwd["op"])[:, None]
    d = out - gt
    g = scale * 2 * d / (3 * n)
    go = -bg * g.sum(1)
    ref = np_composite_f64(sig, rgbs, deltas, ts, rays_a, 1e-4, go, z, g, np.zeros(S))
    return fwd, out, d, ref


def _head_call(lib, t_in, n, half, loss_scale, scale_dev):
    sig, rgbs, dl, ra, gt = t_in
    S = sig.numel()
    loss_sum, op, rgb = torch.zeros(1, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, 3, device=DEV)
    dsig = torch.full((S,), 9.0, device=DEV)
    drgbs = torch.full((S, 3), 9.0, device=DEV, dtype=torch.float16 if half else torch.float32)
    chk(lib.ngp_ray_head_fused(P(sig), P(rgbs), F16 if half else F32, P(dl), P(ra), P(gt), 1.0, loss_scale,
                               P(scale_dev), 1e-4, P(loss_sum), P(op), P(rgb), P(dsig), P(drgbs), n, ST()))
    return loss_sum, op, rgb, dsig, drgbs


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
def test_ray_head_fused_long_rays_fp64(lib, half):
    """gt = 0 and colours in [0, 0.5] with a white background keep every sum sign-coherent, so the tolerance is the
    plain N u sum |terms| bound."""
    rng = np.random.default_rng(71 + half)
    rays_a, sig, rgbs, deltas, ts = _long_rays(rng, half)
    n = rays_a.shape[0]
    gt = np.zeros((n, 3), np.float32)
    scale = 2.0 ** 16
    fwd, out, d, ref = _head_ref(rays_a, sig, rgbs, deltas, ts, gt, 1.0, scale)
    ls, op, rgb, dsig, drgbs = _head_call(lib, [T(a) for a in (sig, rgbs, deltas, rays_a, gt)], n, half, scale, None)
    k = fwd["kray"]
    assert (np.abs(N(op) - fwd["op"]) <= 8 * k * U * fwd["op"] + 1e-30).all()
    assert (np.abs(N(rgb) - out) <= 8 * k[:, None] * U * (out + 2)).all()
    assert abs(float(ls) - (d ** 2).sum()) <= 16 * k.max() * U * (d ** 2).sum()
    _check_composite_bwd(N(dsig), N(drgbs), ref, half, "ray_head_fused")


@pytest.mark.gpu
@pytest.mark.parametrize("s", [2.0 ** -4, 1.0, 2.0 ** 16, 2.0 ** 19, 2.0 ** 24])
def test_device_loss_scale_equals_host_scale(lib, s):
    """scale_dev holding s == the host constant s, bit for bit, for the power-of-two scales GradScaler uses
    (device: (2/(3n))*s, host: (s*2)/(3n)).  loss_sum does not depend on the scale; its atomic order may differ
    between launches, so it is checked against fp64."""
    rng = np.random.default_rng(81)
    rays_a, sig, rgbs, deltas, ts = _long_rays(rng, True)
    n = rays_a.shape[0]
    gt = rng.random((n, 3)).astype(np.float32)
    t_in = [T(a) for a in (sig, rgbs, deltas, rays_a, gt)]
    a = _head_call(lib, t_in, n, True, s, None)
    b = _head_call(lib, t_in, n, True, 12345.0, torch.tensor([s], device=DEV))
    for x, y, name in zip(a[1:], b[1:], ("opacity", "rgb", "dsigma", "drgb")):
        assert torch.equal(x, y), f"s={s}: ray_head_fused {name}"
    assert abs(float(a[0]) - float(b[0])) <= 1e-6 * float(a[0])

    # the separate loss head
    nr = 1037
    rgb = rng.random((nr, 3)).astype(np.float32)
    op = rng.random(nr).astype(np.float32)
    gt = rng.random((nr, 3)).astype(np.float32)
    t_rgb, t_op, t_gt = T(rgb), T(op), T(gt)
    for bg in (0.0, 1.0):
        res = []
        for dev_scale in (None, torch.tensor([s], device=DEV)):
            ls, gr, go = torch.zeros(1, device=DEV), torch.zeros(nr, 3, device=DEV), torch.zeros(nr, device=DEV)
            if dev_scale is None:
                chk(lib.ngp_mse_loss_grad(P(t_rgb), P(t_op), P(t_gt), bg, s, P(ls), P(gr), P(go), nr, ST()))
            else:
                chk(lib.ngp_mse_loss_grad_dyn(P(t_rgb), P(t_op), P(t_gt), bg, P(dev_scale), P(ls), P(gr), P(go),
                                              nr, ST()))
            res.append((ls, gr, go))
        assert torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2]), f"s={s} bg={bg}"
        diff = rgb.astype(np.float64) + bg * (1 - op.astype(np.float64))[:, None] - gt
        terms = np.abs(rgb) + bg * (1 + np.abs(op))[:, None] + np.abs(gt)
        coef = s * 2 / (3 * nr)
        g_ref = coef * diff
        assert (np.abs(N(res[0][1]) - g_ref) <= 8 * U * coef * terms).all()
        go_ref = -bg * g_ref.sum(1)
        assert (np.abs(N(res[0][2]) - go_ref) <= 12 * U * coef * bg * terms.sum(1)).all()
        for ls, _, _ in res:
            assert abs(float(ls) - (diff ** 2).sum()) <= nr * 8 * U * (terms ** 2).sum()


# ---- 7. argument validation (CPU: rejected before any launch) ----------------------------------------------------
def test_step_kernel_argument_validation_needs_no_gpu(lib):
    fake = C.c_void_p(0x10000)
    lay = make_hash_layout(2 ** 19, 16, 16, 1024, 2).as_ctypes()
    bw = lib.ngp_hash_encode_bwd_levels
    for a, b in ((3, 3), (5, 2), (0, 17), (15, 17)):
        assert bw(fake, fake, F32, C.byref(lay), fake, 8, None, None, a, b, None, None) < 0, (a, b)
        assert b"level range" in lib.ngp_last_error()
    lay4 = make_hash_layout(2 ** 19, 4, 16, 1024, 4).as_ctypes()
    assert bw(fake, fake, F32, C.byref(lay4), fake, 8, None, None, 0, 3, None, None) < 0
    assert b"feature_per_level" in lib.ngp_last_error()
    assert bw(fake, fake, F32, C.byref(lay4), fake, 8, None, None, 1, 4, None, None) < 0

    upd = lib.ngp_loss_scale_update
    for growth, backoff, interval in ((0.5, 0.5, 2000), (2.0, 0.0, 2000), (2.0, -0.5, 2000), (2.0, 1.5, 2000),
                                      (2.0, 0.5, 0), (2.0, 0.5, -3)):
        assert upd(fake, fake, growth, backoff, interval, 1.0, fake, 0, None) < 0, (growth, backoff, interval)
        assert b"GradScaler" in lib.ngp_last_error()

    assert lib.ngp_adam_step_dyn(fake, fake, fake, fake, None, None, None, B1, B2, EPS, 1, 8, None) < 0
    assert b"null" in lib.ngp_last_error()
    mis = C.c_void_p(0x10004)
    assert lib.ngp_adam_step_dyn(mis, fake, fake, fake, None, None, fake, B1, B2, EPS, 1, 8, None) < 0
    assert lib.ngp_adam_step_dyn(fake, fake, fake, fake, C.c_void_p(0x10002), None, fake, B1, B2, EPS, 1, 8, None) < 0
    assert lib.ngp_adam_step_dyn_g16(fake, C.c_void_p(0x10002), fake, fake, fake, None, None, fake, B1, B2, EPS, 8,
                                     None) < 0
    assert lib.ngp_adam_step_dyn_g16(fake, fake, mis, fake, fake, None, None, fake, B1, B2, EPS, 8, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert lib.ngp_grad_pack_f16(mis, fake, 8, None) < 0
    assert lib.ngp_grad_pack_f16(fake, C.c_void_p(0x10002), 8, None) < 0
    assert lib.ngp_check_finite_f16(C.c_void_p(0x10008), 8, fake, None) < 0
    assert lib.ngp_check_finite(mis, 8, fake, None) < 0
    assert b"aligned" in lib.ngp_last_error()

    # n = 0: a successful no-op, whatever the pointers
    assert lib.ngp_adam_step_dyn(None, None, None, None, None, None, None, B1, B2, EPS, 1, 0, None) == 0
    assert lib.ngp_adam_step_dyn_g16(None, None, None, None, None, None, None, None, B1, B2, EPS, 0, None) == 0
    assert lib.ngp_grad_pack_f16(None, None, 0, None) == 0
    assert lib.ngp_check_finite_f16(None, 0, None, None) == 0
    assert lib.ngp_check_finite(None, 0, None, None) == 0
    assert bw(None, None, F16, C.byref(lay), None, 0, None, None, 0, 16, None, None) == 0
    assert lib.ngp_mse_loss_grad(None, None, None, 1.0, 1.0, None, None, None, 0, None) == 0
    assert lib.ngp_mse_loss_grad_dyn(None, None, None, 1.0, None, None, None, None, 0, None) == 0
    assert lib.ngp_ray_head_fused(None, None, F16, None, None, None, 1.0, 1.0, None, 1e-4, None, None, None, None,
                                  None, 0, None) == 0
