"""The fused MLP kernels (csrc/mlp.cu) at trained-model magnitudes: the TruncExp clamp, fp16 overflow of a layer output,
sigmoid saturation and fp32 embeddings beyond the fp16 range.

The inputs come from `mlp_tolerance.trained_inputs` (dedicated weight paths put chosen rows in each regime, and the
generator's self-check says they are there); the reference is `mlp_tolerance.autocast_ref`, a float64 restatement of the
autocast graph with IEEE inf / NaN arithmetic.  Per row and output the value class (finite / 0 / 1 / +inf / -inf / NaN)
must be the restatement's; finite elements keep the bounds of the oracle comparisons in test_gpu_parity.py.  On the
"probe" rows (drgb = 0) the TruncExp gradient reaches dL/demb untouched, so dL/de0 = 2 r16(dsig exp(clamp(h0, -15, 15)))
can be asserted exactly where h0 is clamped.  The CPU tests at the end check the restatement against the CPU oracle and
show that the assertions reject the kernel mistakes they are there for."""
import ctypes as C
import functools

import numpy as np
import pytest

from mlp_tolerance import (FINITE_REGIMES, NONFINITE_REGIMES, autocast_ref, check_trained_regimes, h0_reference, r16,
                           trained_inputs, ulp16)

DEV = "cuda"
# tile edges of the 64-row kernels: one row, one tile +-1, two tiles + 1, and every CTA of an H100 (148 SMs x 3) busy
SIZES = [1, 63, 64, 65, 129, 148 * 3 * 64 + 1]
CLASS_NAMES = ("finite", "zero", "one", "+inf", "-inf", "nan")


def classes(x):
    """Value class of every element: 0 finite (not 0 / 1), 1 exactly 0, 2 exactly 1, 3 +inf, 4 -inf, 5 NaN."""
    x = np.asarray(x, np.float64)
    c = np.zeros(x.shape, np.int8)
    c[x == 0] = 1
    c[x == 1] = 2
    c[x == np.inf] = 3
    c[x == -np.inf] = 4
    c[np.isnan(x)] = 5
    return c


def check_classes(name, got, want):
    cg, cw = classes(got), classes(want)
    bad = np.argwhere(cg != cw)
    assert len(bad) == 0, (f"{name}: {len(bad)} elements of another value class, first at {tuple(bad[0])}: kernel "
                           f"{CLASS_NAMES[cg[tuple(bad[0])]]} ({got[tuple(bad[0])]}), reference "
                           f"{CLASS_NAMES[cw[tuple(bad[0])]]} ({want[tuple(bad[0])]})")


def check_probe_rows(demb, sigma, dsig, rows):
    """dL/dh0 on the probe rows, read back from dL/de0 (h0 > 0 rows) or dL/de1 (h0 < 0 rows): 2 r16(dsig exp(c)) with
    c = clamp(h0, -15, 15) and h0 the kernel's own fp16 h0 (recovered from its sigma).  Exact where h0 is clamped -
    exp(+-15) is one fp32 value and dsig is chosen so that the fp32 product is far from an fp16 rounding boundary;
    within one ulp16 elsewhere (exp(h0) in fp32 may differ in its last bit).  Returns the number of clamped rows."""
    r = rows["probe"]
    with np.errstate(divide="ignore"):
        h0 = r16(np.log(np.asarray(sigma, np.float64)[r]))
    c = np.clip(h0, -15.0, 15.0)
    ds = r16(np.float32(dsig[r]) * np.exp(np.float32(c)))
    pos = np.isin(r, np.concatenate([rows[k] for k in ("h0_gt15", "h0_near+15", "h0_8to11")]))
    got = np.where(pos, demb[r, 0], demb[r, 1]).astype(np.float64)
    want = np.where(pos, 2 * ds, -2 * ds)
    clamped = np.abs(h0) >= 15
    assert np.isfinite(h0).all() and ((h0 > 0) == pos).all(), (r, h0)
    assert (got[clamped] == want[clamped]).all(), \
        ("TruncExp backward at the clamp", r[clamped], h0[clamped], got[clamped], want[clamped])
    tol = ulp16(want[~clamped])
    assert (np.abs(got[~clamped] - want[~clamped]) <= tol).all(), \
        ("TruncExp backward", r[~clamped], h0[~clamped], got[~clamped], want[~clamped])
    return int(clamped.sum())


def check_finite_bounds(sig, rgb, demb, ref, emb, ws):
    """The oracle comparisons' bounds on the elements finite in both: h0 within the fp16 flip bound of
    mlp_tolerance.h0_reference, rgb within 2e-3, dL/demb 99.9th percentile within 1e-4 and every element within 5e-3 of
    the largest reference magnitude.  Returns (max h0 error in ulp16, max rgb error, max demb error / max)."""
    fin = np.isfinite(ref["sigma"]) & (ref["sigma"] > 0) & np.isfinite(sig) & (sig > 0)
    out = [0.0, 0.0, 0.0]
    if fin.any():
        e = np.asarray(emb, np.float32)[fin]
        _, bound = h0_reference(e, ws)
        err = np.abs(np.log(sig[fin].astype(np.float64)) - np.log(ref["sigma"][fin]))
        assert (err <= bound + 4e-7 * (1 + np.abs(ref["h0"][fin]))).all(), np.max(err - bound)
        out[0] = float((err / ulp16(ref["h0"][fin])).max())
    f = np.isfinite(rgb) & np.isfinite(ref["rgb"])
    if f.any():
        out[1] = float(np.abs(rgb[f] - ref["rgb"][f]).max())
        assert out[1] <= 2e-3, out[1]
    if demb is not None:
        f = np.isfinite(demb) & np.isfinite(ref["demb"])
        if f.any():
            err, m = np.abs(demb[f] - ref["demb"][f]), np.abs(ref["demb"][f]).max()
            assert np.percentile(err, 99.9) <= 1e-4 * m and err.max() <= 5e-3 * m, (np.percentile(err, 99.9), err.max(), m)
            out[2] = float(err.max() / max(m, 1e-30))
    return out


@functools.lru_cache(maxsize=None)
def _case(n, emb_half, seed=11):
    emb, dirs, ws, dsig, drgb, rows = trained_inputs(n, seed, np.float16 if emb_half else np.float32, finite=False)
    ref = autocast_ref(emb, dirs, ws, dsig, drgb)
    check_trained_regimes(ref, rows)
    return emb, dirs, ws, dsig, drgb, rows, ref


def _T(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _N(t):
    return t.detach().float().cpu().numpy()


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("saved", [False, True])
@pytest.mark.parametrize("emb_half", [True, False])
@pytest.mark.parametrize("n", SIZES)
def test_trained_rows_match_autocast_restatement(n, emb_half, saved):
    """Every regime of trained_inputs (TruncExp clamp on both sides and at +-15 +- ulp, |h0| in 8..11, fp16 sigmoid
    exactly 0 / 1, overflow of layers 1 / 3 / 4, of exp(h0) and of h0 itself, dL/demb overflow), special rows at the
    first / last row and on both sides of 64-row tile edges: forward and both backward paths (recompute; restart from
    the saved h and fp16 rgb, kSaved) against the float64 restatement, value class by value class."""
    from taichi_nerfs_b200 import ops
    emb, dirs, ws, dsig, drgb, rows, ref = _case(n, emb_half)
    tw = [_T(w) for w in ws]
    sig, rgb, save = ops.mlp_fwd(_T(emb), _T(dirs), tw, with_save=True)
    demb, gw = ops.mlp_bwd(_T(emb), _T(dirs), tw, _T(dsig), _T(drgb), save=save if saved else None)
    sig, rgb, demb, gw = _N(sig), _N(rgb), _N(demb), _N(gw)
    check_classes("sigma", sig, ref["sigma"])
    check_classes("rgb", rgb, ref["rgb"])
    check_classes("dL/demb", demb, ref["demb"])
    errs = check_finite_bounds(sig, rgb, demb, ref, emb, ws)
    clamped = check_probe_rows(demb, sig, dsig, rows)
    special = np.concatenate([v for k, v in rows.items() if k != "probe"])
    nonfin = ~np.isfinite(demb).all(1)
    print(f"n={n} emb={'f16' if emb_half else 'f32'} saved={saved}: {len(special)} special rows, {clamped} clamped "
          f"probe rows, {int(nonfin.sum())} rows with non-finite dL/demb; max h0 err {errs[0]:.2f} ulp16, rgb "
          f"{errs[1]:.2e}, demb {errs[2]:.2e} of max")
    # a non-finite dL/demb comes with a non-finite weight gradient except on the dL/demb-overflow rows
    if nonfin.any() and not np.isin(np.nonzero(nonfin)[0], rows["demb_overflow"]).all():
        assert not np.isfinite(gw).all()


def _dyn(emb, dirs, ws, dsig, drgb, n_dev, cap_pad):
    """Forward and backward through the device-count entries, outputs pre-filled with a sentinel; found_inf given."""
    import torch
    from taichi_nerfs_b200 import _lib, ops
    lib = _lib.load()
    cap = emb.shape[0]
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    te, td, tds, tdr = _T(emb), _T(dirs), _T(dsig), _T(drgb)      # held until the launches are done
    tag = _lib.F16 if emb.dtype == np.float16 else _lib.F32
    w, keep = ops._mlp_weights([_T(x) for x in ws])
    sig = torch.full((cap + cap_pad,), -7.0, device=DEV)
    rgb = torch.full((cap + cap_pad, 3), -7.0, device=DEV, dtype=torch.float16)
    save = torch.zeros(int(lib.ngp_mlp_save_bytes(cap)), device=DEV, dtype=torch.uint8)
    nd = torch.tensor([n_dev], device=DEV, dtype=torch.int32)
    _lib.check(lib.ngp_mlp_fwd_dyn(p(te), tag, p(td), C.byref(w), p(sig), p(rgb), p(save), cap, p(nd), st))
    demb = torch.full((cap + cap_pad, 32), -7.0, device=DEV, dtype=te.dtype)
    gw = torch.zeros(9408, device=DEV)
    found = torch.zeros(1, device=DEV, dtype=torch.int32)
    _lib.check(lib.ngp_mlp_bwd_dyn(p(te), tag, p(td), C.byref(w), p(save), p(tds), p(tdr), p(demb), p(gw),
                                   cap, p(nd), p(found), st))
    torch.cuda.synchronize()
    return _N(sig), _N(rgb), _N(demb), _N(gw), int(found.item())


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["in", "beyond"])
@pytest.mark.parametrize("kind", ["none", "l1_overflow", "l3_overflow", "l4_overflow", "h0_f16_overflow",
                                  "h0_exp_overflow", "demb_overflow"])
def test_found_inf_from_inside_the_mlp(kind, where):
    """found_inf of ngp_mlp_bwd_dyn is raised iff its weight gradient or dL/demb (rows below the device count) holds a
    non-finite value, with the non-finite value arising inside the MLP: a layer that overflows fp16 in the forward, or
    dL/demb overflowing in its last rounding while every weight gradient stays finite ("demb_overflow", which reaches
    the dL/demb check alone).  exp(h0) overflowing gives sigma = inf but finite gradients: no flag.  One special row
    inside the device count or beyond it; rows past n_dev keep the sentinel in every output."""
    cap, n_dev = 4000, 3000
    emb, dirs, ws, dsig, drgb, _ = trained_inputs(cap, 5, finite=True)
    row = {"in": 1234, "beyond": 3500}[where]
    if kind != "none":
        from mlp_tolerance import _regime_row
        e, dsig[row], drgb[row] = _regime_row(kind, 0, np.random.default_rng(3))
        emb[row] = e.astype(np.float16)
    sig, rgb, demb, gw, flag = _dyn(emb, dirs, ws, dsig, drgb, n_dev, 0)
    ref = autocast_ref(emb[:n_dev], dirs[:n_dev], ws, dsig[:n_dev], drgb[:n_dev])
    check_classes("sigma", sig[:n_dev], ref["sigma"])
    check_classes("rgb", rgb[:n_dev], ref["rgb"])
    check_classes("dL/demb", demb[:n_dev], ref["demb"])
    bad = not (np.isfinite(gw).all() and np.isfinite(demb[:n_dev]).all())
    assert flag == int(bad), f"found_inf={flag}, non-finite weight gradient or dL/demb: {bad}"
    expect = where == "in" and kind not in ("none", "h0_exp_overflow")
    assert flag == int(expect)
    if kind == "demb_overflow" and where == "in":
        assert np.isfinite(gw).all() and not np.isfinite(demb[row]).all()
    if kind == "h0_exp_overflow" and where == "in":
        assert sig[row] == np.inf
    assert (sig[n_dev:] == -7).all() and (rgb[n_dev:] == -7).all() and (demb[n_dev:] == -7).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [65, 148 * 3 * 64 + 1])
def test_rows_past_device_count_untouched(n):
    """Every regime inside [0, n_dev) of a larger buffer, n_dev on a tile edge + 1: rows past n_dev and the padding
    keep the sentinel in sigma, rgb and dL/demb; rows below it are what the host-count launch gives."""
    from taichi_nerfs_b200 import ops
    emb, dirs, ws, dsig, drgb, rows, ref = _case(n, True)
    cap, pad = n + 200, 64
    rng = np.random.default_rng(1)
    big = lambda a, fill: np.concatenate([a, fill(cap - n)]).astype(a.dtype)  # noqa: E731
    e2 = big(emb, lambda k: rng.standard_normal((k, 32)))
    sig, rgb, demb, gw, flag = _dyn(e2, big(dirs, lambda k: rng.standard_normal((k, 3))), ws, big(dsig, np.ones),
                                    big(drgb, lambda k: np.ones((k, 3))), n, pad)
    tw = [_T(w) for w in ws]
    s_ref, r_ref = ops.mlp_fwd(_T(emb), _T(dirs), tw)
    assert np.array_equal(sig[:n], _N(s_ref), equal_nan=True) and np.array_equal(rgb[:n], _N(r_ref), equal_nan=True)
    check_classes("dL/demb", demb[:n], ref["demb"])
    assert flag == 1
    assert (sig[n:] == -7).all() and (rgb[n:] == -7).all() and (demb[n:] == -7).all()


@pytest.mark.gpu
@pytest.mark.parametrize("saved", [False, True])
def test_fp32_embeddings_beyond_fp16_range(saved):
    """The tri-plane model feeds fp32 features; load_emb's conversion must round them like autocast's cast: 65519 to
    65504, 65520 and above to inf.  The fp32 path then gives exactly what the fp16 path gives when fed those fp16
    values (inf included), in every output."""
    from taichi_nerfs_b200 import ops
    n = 300
    emb, dirs, ws, dsig, drgb, rows = trained_inputs(n, 17, np.float32, finite=True)
    big = {0: (4, 1e5), 63: (5, -1e5), 64: (6, 65519.0), 129: (7, 65520.0), 130: (8, -65520.0), 299: (9, 3e38)}
    for r, (k, v) in big.items():
        emb[r, k] = v
    with np.errstate(over="ignore"):
        e16 = emb.astype(np.float16)
    assert np.isinf(e16[[0, 63, 129, 130, 299]]).any(1).all() and e16[64, 6] == 65504
    ref = autocast_ref(emb, dirs, ws, dsig, drgb)
    tw = [_T(w) for w in ws]
    out = {}
    for name, e in (("f32", emb), ("f16", e16)):
        sig, rgb, save = ops.mlp_fwd(_T(e), _T(dirs), tw, with_save=True)
        demb, gw = ops.mlp_bwd(_T(e), _T(dirs), tw, _T(dsig), _T(drgb), save=save if saved else None)
        out[name] = [_N(sig), _N(rgb), _N(demb), _N(gw)]
    for a, b, what in zip(out["f32"], out["f16"], ("sigma", "rgb", "dL/demb", "weight gradient")):
        if what == "weight gradient":   # fp32 atomics: the order of the per-CTA flushes may differ between launches
            check_classes(what, a, b)
        else:
            assert np.array_equal(a, b, equal_nan=True), what
    check_classes("sigma", out["f32"][0], ref["sigma"])
    check_classes("rgb", out["f32"][1], ref["rgb"])
    check_classes("dL/demb", out["f32"][2], ref["demb"])
    assert not np.isfinite(out["f32"][3]).all()      # inf in E reaches dW1 = dH1^T E


# ---- CPU: the restatement and the assertions themselves -------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("finite", [True, False])
def test_trained_inputs_reach_every_regime(n, finite):
    """The generator's rows are in their regimes at every size; with room for them, every regime has its rows, and the
    finite ones give finite outputs and gradients."""
    emb, dirs, ws, dsig, drgb, rows = trained_inputs(n, 11, finite=finite)
    ref = autocast_ref(emb, dirs, ws, dsig, drgb)
    got = check_trained_regimes(ref, rows)
    kinds = FINITE_REGIMES + (() if finite else NONFINITE_REGIMES)
    if n >= 6 * len(kinds):
        assert set(got) == set(kinds) and min(got.values()) == 6, got
    if finite:
        assert all(np.isfinite(ref[k]).all() for k in ("sigma", "rgb", "demb"))


@pytest.mark.parametrize("emb_half", [True, False])
def test_restatement_matches_oracle(oracle, emb_half):
    """On finite rows the float64 restatement and the CPU oracle agree within the oracle comparisons' bounds, and the
    oracle passes the exact TruncExp-clamp check too."""
    emb, dirs, ws, dsig, drgb, rows = trained_inputs(2000, 23, np.float16 if emb_half else np.float32, finite=True)
    ref = autocast_ref(emb, dirs, ws, dsig, drgb)
    sig, rgb = oracle.mlp_fwd(emb, dirs, ws)
    demb, _ = oracle.mlp_bwd(emb, dirs, ws, dsig, drgb)
    sig, rgb, demb = sig.astype(np.float64), rgb.astype(np.float64), demb.astype(np.float64)
    for name, a, b in (("sigma", sig, ref["sigma"]), ("rgb", rgb, ref["rgb"]), ("dL/demb", demb, ref["demb"])):
        check_classes(name, a, b)
    check_finite_bounds(sig, rgb, demb, ref, emb, ws)
    assert check_probe_rows(demb, sig, dsig, rows) > 0
    assert check_probe_rows(ref["demb"], ref["sigma"], dsig, rows) > 0


FAULTS = ["no_clamp", "clamp_hi_only", "clamp_unrounded", "sat_unrounded"]


@pytest.mark.parametrize("fault", FAULTS)
def test_assertions_reject_seeded_faults(fault):
    """A restated kernel with one mistake fails the assertions the GPU tests make: the TruncExp clamp removed, applied
    at +15 only, or applied to the unrounded h0 (the probe-row check), and the sigmoid backward taken as y (1 - y) in
    fp32 on the unrounded y (the value-class check: a saturated channel's gradient must vanish)."""
    emb, dirs, ws, dsig, drgb, rows = trained_inputs(2000, 31, finite=True)
    good = autocast_ref(emb, dirs, ws, dsig, drgb)
    bad = autocast_ref(emb, dirs, ws, dsig, drgb, fault=fault)
    check_probe_rows(good["demb"], good["sigma"], dsig, rows)
    with pytest.raises(AssertionError):
        check_probe_rows(bad["demb"], bad["sigma"], dsig, rows)
        check_classes("dL/demb", bad["demb"], good["demb"])
