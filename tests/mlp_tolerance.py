"""Per-element error model for the fused MLP forward (north_star: sigma / rgb within 1e-3 fp16 relative).

Both sides (CUDA kernels, oracle) use fp16 operands, fp32 accumulation and round every layer output to fp16; the
tensor core adds the K products in a different order than the oracle's sequential loop, so two fp32 sums that straddle
an fp16 rounding boundary round to NEIGHBOURING fp16 values ("flip", 1 ulp).  Consequences for h0 = (relu(E W1^T) W2^T)[0]
(sigma = exp(h0), so |d sigma| / sigma = |d h0|):

  * own rounding of h0: <= 1 ulp16(h0);
  * every H1 element may flip by one ulp16(H1_k) <= 2^-10 |H1_k|, which moves the fp32 sum by |W2[0,k]| ulp16(H1_k):
    worst case sum_k |W2[0,k]| ulp16(H1_k)  (all 64 elements flipping the same way - the rigorous bound);
  * in practice flips are rare (a sum must land within ~1e-6 relative of a boundary): the typical error is 0 ulp.

`h0_bound` returns the rigorous per-element bound; the tests assert it for every element and, separately, that the
99th percentile stays within 2 ulp16(h0) (= 1e-3 relative on sigma for |h0| < 1) and the median is exact.
"""
import numpy as np


def ulp16(x):
    """Spacing of fp16 at |x| (normal range; subnormal spacing 2^-24 below 2^-14)."""
    a = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


def h0_reference(emb, ws):
    """(h0 as fp16-rounded float64, rigorous flip bound) from an independent numpy restatement of layers 1-2."""
    e = np.asarray(emb, np.float16).astype(np.float32)
    w1 = ws[0].astype(np.float16).astype(np.float32)
    w2 = ws[1].astype(np.float16).astype(np.float32)
    h1 = np.maximum(e @ w1.T, 0).astype(np.float16).astype(np.float32)
    h0 = (h1 @ w2[0]).astype(np.float16).astype(np.float64)
    flip = (np.abs(w2[0])[None, :].astype(np.float64) * np.where(h1 > 0, ulp16(h1), 0.0)).sum(1)
    return h0, ulp16(h0) + flip


def check_sigma(sig_got, sig_ref, emb, ws):
    h_ref = np.log(np.asarray(sig_ref, np.float64))
    h_got = np.log(np.asarray(sig_got, np.float64))
    h_np, bound = h0_reference(emb, ws)
    err = np.abs(h_got - h_ref)
    slack = 4e-7 * (1 + np.abs(h_ref))          # log/exp round trip in fp32
    assert (err <= bound + slack).all(), f"max excess {np.max(err - bound):.3e}"
    # the independent numpy restatement agrees with the oracle under the same model
    assert (np.abs(h_np - h_ref) <= bound + slack).all()
    u = err / ulp16(h_ref)
    assert np.percentile(u, 99) <= 2.0 + 1e-3, np.percentile(u, 99)
    assert np.median(u) <= 1e-3
    return float(u.max())


# ---- trained-model magnitudes ----------------------------------------------------------------------------------------
# Xavier weights and standard-normal embeddings keep h0 near O(1), every hidden activation far below the fp16 limit and
# every sigmoid away from 0 / 1.  A trained NeRF does not: empty space drives h0 below -15, surfaces above it, and late
# in training the rgb logits saturate.  `trained_inputs` builds weights with a few dedicated paths (the rest Xavier) so
# that chosen rows land in each of those regimes, and `autocast_ref` restates the autocast graph in float64 (every
# nn.Linear output rounded to fp16, ReLU on the rounded value, TruncExp and sigmoid in fp32, gradients rounded to fp16
# where autocast rounds them) with IEEE inf / NaN arithmetic, so it also says what a non-finite row must give.
#
# Dedicated paths (emb coordinates c0..c3, everything else Xavier):
#   h0 = 2 relu(e0) - 2 relu(e1) + relu(4 e3) + (Xavier part over H1[5:])      W1 rows 0, 1, 4; W2 row 0
#   h1 = relu(e2) - relu(-e2) + (Xavier part / 32)                              W1 rows 2, 3; W2 row 1
#   H3[0] = relu(4 h1), H3[1] = relu(-4 h1), H4[0] = relu(4 H3[0]), H4[1] = relu(4 H3[1])
#   o0 = H4[0] - H4[1] + (Xavier part / 32),  o1 = -o0 + ...,  o2 Xavier
# so e0 / e1 place h0, e2 places the rgb logits (o0 ~ 16 e2) or overflows layer 3 / 4, and e3 overflows layer 1.
# On a "probe" row (drgb = 0) dL/dh is [ds, 0, ...] with ds = r16(dsig exp(clamp(h0))), and it reaches dL/demb exactly:
# dL/de0 = 2 ds (h0 = 2 e0 + ...) and dL/de1 = -2 ds.
F16_MAX = 65504.0
EXP15 = float(np.exp(np.float32(15.0)))
EXPM15 = float(np.exp(np.float32(-15.0)))

# finite regimes (used by the oracle comparisons) and non-finite ones (tests/test_gpu_mlp_magnitudes.py)
FINITE_REGIMES = ("h0_gt15", "h0_lt-15", "h0_near+15", "h0_near-15", "h0_8to11", "h0_-11to-8", "rgb_sat1", "rgb_sat0")
NONFINITE_REGIMES = ("l1_overflow", "l3_overflow", "l4_overflow", "h0_exp_overflow", "h0_f16_overflow",
                     "h0_f16_overflow_neg", "demb_overflow")


def r16(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def trained_weights(rng):
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    w1, w2, w3, w4, w5 = [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))) for s in shapes]
    u = np.eye(64)
    w1[:, :4] = 0
    w1[0], w1[1], w1[2], w1[3], w1[4] = u[0, :32], u[1, :32], u[2, :32], -u[2, :32], 4 * u[3, :32]
    w2[0, :5] = [2, -2, 0, 0, 1]
    w2[1, :4] = [0, 0, 1, -1]
    w2[1, 4:] /= 32
    w2[2:, 2:4] = 0
    w3[2:, 16] /= 64
    w3[:, 17] = 0
    w3[0], w3[1] = 4 * u[17, :32], -4 * u[17, :32]
    w4[:, :2] = 0
    w4[0], w4[1] = 4 * u[0], 4 * u[1]
    w5[:2, 2:] /= 32
    w5[:, :2] = [[1, -1], [-1, 1], [0, 0]]
    return [w.astype(np.float32) for w in (w1, w2, w3, w4, w5)]


def _regime_row(kind, j, rng):
    """(emb row as float64, dsig, drgb) for the j-th special row of regime `kind`."""
    e = np.zeros(32)
    e[4:] = rng.standard_normal(28)
    e[2] = rng.standard_normal() * 0.05
    dsig, drgb = 0.0, np.zeros(3)
    s = rng.choice([-1.0, 1.0])
    if kind == "h0_gt15":      # clamped at +15: ds = r16(dsig exp(15)) = target exactly
        e[0] = rng.uniform(9.5, 20)
        dsig = rng.choice([0.25, 3.0, 1000.0]) / EXP15
    elif kind == "h0_lt-15":
        e[1] = rng.uniform(9.5, 20)
        dsig = rng.choice([2.0 ** -10, 0.25, 3.0]) / EXPM15
    elif kind in ("h0_near+15", "h0_near-15"):   # h0 within an ulp16 (2^-7 below 16) of +-15: tiny Xavier part
        # e[4:] = 0 leaves h0 = +-2 e + 4 e3 exactly; |h0| before rounding is 15 -+ 2^-9 (rounds to 15 from either
        # side) or 15 +- (2^-7 - 2^-9) (rounds to 15 +- ulp16)
        e[4:] = 0
        de, e3 = ([-1, 0, 1, -1], [3, 1, 1, 1]) if kind == "h0_near+15" else ([0, 1, 1, -1], [1, 3, 1, 1])
        e[0 if kind == "h0_near+15" else 1] = 7.5 + 2.0 ** -8 * de[j % 4]
        e[3] = 2.0 ** -11 * e3[j % 4]
        dsig = 0.5 / EXP15 * rng.uniform(0.5, 2) if kind == "h0_near+15" else 0.5 / EXPM15 * rng.uniform(0.5, 2)
    elif kind in ("h0_8to11", "h0_-11to-8"):      # ulp16(h0) = 2^-7: an unrounded h0 shows as up to ~1 % in exp
        e[0 if kind == "h0_8to11" else 1] = 4.75
        e[4:] *= 0.25
        dsig = rng.uniform(0.5, 2) * np.exp(-9.5 if kind == "h0_8to11" else 9.5)
    elif kind == "rgb_sat1":   # o ~ +-12: fp16 sigmoid exactly 1 (fp32 not), the other channel not saturated
        e[2] = 0.75 * s
        drgb[0 if s > 0 else 1] = rng.choice([-100.0, 100.0])
    elif kind == "rgb_sat0":   # o ~ -+20: fp16 sigmoid exactly 0 (fp32 not), the other channel exactly 1
        e[2] = 1.25 * s
        drgb[:2] = rng.choice([-100.0, 100.0], 2)
    elif kind == "l1_overflow":
        e[3] = 30000.0
    elif kind == "l3_overflow":
        e[2] = 30000.0 * s
    elif kind == "l4_overflow":
        e[2] = 5000.0 * s
    elif kind == "h0_exp_overflow":   # finite fp16 h0 above 88.7: sigma = inf, gradients finite
        e[0] = 50.0
        dsig = 1e-3
    elif kind == "h0_f16_overflow":
        e[0] = 40000.0
    elif kind == "h0_f16_overflow_neg":
        e[1] = 40000.0
    elif kind == "demb_overflow":   # dL/dH1 finite, dL/de3 = 4 dL/dH1[4] = 4 ds > 65504: weight gradients stay finite
        e[0], e[3] = 10.0, 0.5
        dsig = 32000.0 / EXP15
    else:
        raise ValueError(kind)
    if kind not in FINITE_REGIMES[:6] and not kind.startswith("rgb"):
        drgb = rng.standard_normal(3) * 0.1
    return e, dsig, drgb


def special_rows(n):
    """Rows the special cases go to: the first, the last and both sides of every 64-row tile boundary (rows 63 / 64,
    127 / 128, ...), then spread over the rest."""
    cand = [0, n - 1]
    for b in range(64, n, 64):
        cand += [b - 1, b]
    seen, out = set(), []
    for r in cand:
        if 0 <= r < n and r not in seen:
            seen.add(r)
            out.append(r)
    return out


def trained_inputs(n, seed, emb_dtype=np.float16, finite=True, per_regime=6):
    """Weights, embeddings, directions and upstream gradients at trained-model magnitudes.

    Returns (emb, dirs, ws, dsig, drgb, rows) with rows = {regime: row indices}, plus "probe": the rows whose drgb is 0
    and whose dL/dh0 path is exact (see above).  ``finite=True`` uses only FINITE_REGIMES.  Special rows fill the
    tile-edge positions of `special_rows` first; every other row is a Xavier-magnitude row."""
    rng = np.random.default_rng(seed)
    ws = trained_weights(rng)
    emb = rng.standard_normal((n, 32))
    emb[:, :2] = np.abs(emb[:, :2]) * 0.5
    emb[:, 2] *= 0.05
    emb[:, 3] *= 0.1
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    dsig = rng.standard_normal(n) * 0.1
    drgb = rng.standard_normal((n, 3)) * 0.1
    kinds = list(FINITE_REGIMES) + ([] if finite else list(NONFINITE_REGIMES))
    order = special_rows(n)
    extra = [r for r in rng.permutation(n) if r not in set(order)]
    slots = (order + extra)[:min(n, len(kinds) * per_regime)]
    rows = {k: [] for k in kinds}
    for j, r in enumerate(slots):
        k = kinds[j % len(kinds)]
        emb[r], dsig[r], drgb[r] = _regime_row(k, j // len(kinds), rng)
        rows[k].append(int(r))
    rows = {k: np.array(v, np.int64) for k, v in rows.items()}
    rows["probe"] = np.sort(np.concatenate([rows[k] for k in FINITE_REGIMES[:6] if k in rows]))
    emb = emb.astype(np.float16).astype(emb_dtype)
    return emb, dirs, ws, dsig.astype(np.float32), drgb.astype(np.float16), rows


# ---- float64 restatement of the autocast graph ----------------------------------------------------------------------
def _lin(x, w):
    """x [n, k] @ w^T [k, o] with IEEE inf / NaN products (a BLAS call may skip zeros), summed in float64."""
    out = np.empty((x.shape[0], w.shape[0]))
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(0, x.shape[0], 256):
            out[s:s + 256] = (x[s:s + 256, None, :] * w[None]).sum(-1)
    return out


def _relu(x):
    return np.where(x > 0, x, np.where(np.isnan(x), x, 0.0))       # torch.relu keeps NaN


def _relu_bwd(g, act):
    return np.where(act <= 0, 0.0, g)                              # threshold_backward: NaN activations pass


def _sh16(d):
    n = np.sqrt((d * d).sum(1, keepdims=True))
    x, y, z = ((d / n + 1) / 2).T
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    return np.stack([np.full_like(x, 0.28209479177387814), -0.48860251190291987 * y, 0.48860251190291987 * z,
                     -0.48860251190291987 * x, 1.0925484305920792 * xy, -1.0925484305920792 * yz,
                     0.94617469575755997 * z2 - 0.31539156525251999, -1.0925484305920792 * xz,
                     0.54627421529603959 * x2 - 0.54627421529603959 * y2, 0.59004358992664352 * y * (-3 * x2 + y2),
                     2.8906114426405538 * xy * z, 0.45704579946446572 * y * (1 - 5 * z2),
                     0.3731763325901154 * z * (5 * z2 - 3), 0.45704579946446572 * x * (1 - 5 * z2),
                     1.4453057213202769 * z * (x2 - y2), 0.59004358992664352 * x * (-x2 + 3 * y2)], 1)


def _exp32(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.exp(np.asarray(x, np.float32)).astype(np.float64)


def _sigmoid32(o):
    with np.errstate(over="ignore", invalid="ignore"):
        o = np.asarray(o, np.float32)
        return (np.float32(1) / (np.float32(1) + np.exp(-o))).astype(np.float64)


def _clamp(x, lo, hi):
    return np.where(x < lo, lo, np.where(x > hi, hi, x))           # torch.clamp keeps NaN


def autocast_ref(emb, dirs, ws, dsig=None, drgb=None, fault=None):
    """float64 restatement of the autocast MLP.  Returns a dict with sigma, rgb (fp16 values as float64), h0 (rounded),
    h0_raw (fp32 sum before rounding), o (rounded logits), the pre-activations of layers 1 / 3 / 4 and, given dsig /
    drgb, ds (the TruncExp gradient into h0) and demb (fp16-rounded).

    ``fault`` restates a wrong kernel, for the self-checks: "no_clamp", "clamp_hi_only" (clamp at +15 only),
    "clamp_unrounded" (clamp and exp of the unrounded h0) or "sat_unrounded" (sigmoid backward y (1 - y) in fp32 on the
    unrounded y)."""
    e = r16(np.asarray(emb, np.float32))          # the fp16 cast of an fp32 embedding: above 65504 becomes inf
    W = [r16(w) for w in ws]
    p1 = _lin(e, W[0])
    H1 = _relu(r16(p1))
    h_raw = _lin(H1, W[1])
    h = r16(h_raw)
    h0 = h[:, 0]
    x3 = np.concatenate([r16(_sh16(np.asarray(dirs, np.float64))), h], 1)
    p3 = _lin(x3, W[2])
    H3 = _relu(r16(p3))
    p4 = _lin(H3, W[3])
    H4 = _relu(r16(p4))
    o_raw = _lin(H4, W[4])
    o = r16(o_raw)
    y = _sigmoid32(o)
    out = dict(sigma=_exp32(h0), rgb=r16(y), h0=h0, h0_raw=np.asarray(h_raw[:, 0], np.float32).astype(np.float64),
               o=o, p1=r16(p1), p3=r16(p3), p4=r16(p4))
    if dsig is None:
        return out
    rgb = out["rgb"]
    g = np.asarray(drgb, np.float16).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        if fault == "sat_unrounded":
            yu = _sigmoid32(o_raw)
            dO = r16(g * yu * (1 - yu))
        else:
            dO = r16(g * (1 - rgb) * rgb)
        dH4 = _relu_bwd(r16(dO @ W[4] if np.isfinite(dO).all() else _lin(dO, W[4].T)), H4)
        dH3 = _relu_bwd(r16(_lin(dH4, W[3].T)), H3)
        dX3 = r16(_lin(dH3, W[2].T))
        x = out["h0_raw"] if fault == "clamp_unrounded" else h0
        if fault == "no_clamp":
            c = x
        elif fault == "clamp_hi_only":
            c = np.where(x > 15, 15.0, x)
        else:
            c = _clamp(x, -15.0, 15.0)
        ds = r16(np.asarray(dsig, np.float32).astype(np.float64) * _exp32(c))
        dh = dX3[:, 16:].copy()
        dh[:, 0] = r16(dh[:, 0] + ds)
        dH1 = _relu_bwd(r16(_lin(dh, W[1].T)), H1)
        out["ds"] = ds
        out["demb"] = r16(_lin(dH1, W[0].T))
    return out


def check_trained_regimes(ref, rows):
    """The rows `trained_inputs` placed in each regime are there (on the float64 restatement): counts per regime."""
    h0, hr, o, rgb = ref["h0"], ref["h0_raw"], ref["o"], ref["rgb"]
    u15 = 2.0 ** -7                                        # ulp16 in [8, 16)
    got = {}
    for k, r in rows.items():
        if k == "probe" or len(r) == 0:
            continue
        if k == "h0_gt15":
            ok = h0[r] > 15 + u15
        elif k == "h0_lt-15":
            ok = h0[r] < -15 - u15
        elif k in ("h0_near+15", "h0_near-15"):
            sgn = 1 if k == "h0_near+15" else -1
            ok = (np.abs(sgn * h0[r] - 15) <= u15) & (hr[r] != h0[r])
            if len(r) >= 6:
                for v in (15 - u15, 15, 15 + u15):         # both sides of the clamp, and the clamp value itself
                    assert (sgn * h0[r] == v).any(), (k, v, h0[r])
                # rounded h0 = +-15 from an unrounded value inside (-15, 15): clamping the unrounded value shows
                assert ((np.abs(hr[r]) < 15) & (np.abs(h0[r]) == 15)).any(), (k, hr[r])
        elif k in ("h0_8to11", "h0_-11to-8"):
            a = h0[r] * (1 if k == "h0_8to11" else -1)
            ok = (a >= 8) & (a <= 11) & (hr[r] != h0[r])
        elif k == "rgb_sat1":
            ok = (rgb[r] == 1).any(1) & (np.abs(o[r]).max(1) < 16)        # fp16 sigmoid 1, fp32 sigmoid not
        elif k == "rgb_sat0":
            ok = (rgb[r] == 0).any(1) & (rgb[r] == 1).any(1) & (o[r].min(1) > -21.5)
        elif k == "l1_overflow":
            ok = (np.abs(ref["p1"][r]) == np.inf).any(1)
        elif k == "l3_overflow":
            ok = (np.abs(ref["p3"][r]) == np.inf).any(1) & np.isfinite(ref["p1"][r]).all(1)
        elif k == "l4_overflow":
            ok = (np.abs(ref["p4"][r]) == np.inf).any(1) & np.isfinite(ref["p3"][r]).all(1)
        elif k == "h0_exp_overflow":
            ok = (h0[r] > 88.8) & np.isfinite(h0[r]) & (ref["sigma"][r] == np.inf)
        elif k == "h0_f16_overflow":
            ok = h0[r] == np.inf
        elif k == "h0_f16_overflow_neg":
            ok = (h0[r] == -np.inf) & (ref["sigma"][r] == 0)
        elif k == "demb_overflow":
            ok = (np.abs(ref["demb"][r]) == np.inf).any(1) if "demb" in ref else np.ones(len(r), bool)
        assert ok.all(), (k, r[~ok])
        got[k] = len(r)
    return got
