"""References for the tri-plane encoder (csrc/triplane.cu; tests/test_triplane.py, tests/test_gpu_triplane.py,
tests/test_gpu_triplane_fp64.py).

- `triplane_axes`: the per-level geometry in fp32, exactly as sample_axes computes it.
- `triplane_numpy`: the forward, vectorised; bit-exact against the kernel and the oracle in fp32.
- `np_triplane_bwd_f64`: the table backward as an fp64 scatter with its per-float error scale and contribution count;
  `_check_triplane_scatter` holds a kernel's gradient to it with a bound that is valid in any atomic order.

Tables are passed either as an array or as a callable `table_at(float indices) -> values`, so that a table too large
for the host (max_res 16384: 12.9 GB at F = 4) can be described by a function of the element index.
"""
import numpy as np

U = 2.0 ** -24          # fp32 unit roundoff
PLANES = ((0, 1), (1, 2), (2, 0))   # plane fd: (first axis, stride 1), (second axis, stride max_res); triplane.py:46-50
C_TERM = 11             # roundings in one kernel term, see _check_triplane_scatter


def _table_at(table):
    if callable(table):
        return table
    tab = np.asarray(table)
    return lambda e: tab[e]


def triplane_axes(x, lay, level):
    """fp32 geometry of one level for positions x [n, 3], as sample_axes (csrc/triplane.cu) computes it.  Per axis k:
    a[k] = (1 - fr, fr) and q[k] = (f32(g) / res * (max_res-1), f32(g+1) / res * (max_res-1)), the max_res-grid
    coordinates before truncation.  pos = x*(res-1) + 0.5, g = floor(pos) saturated at 0 (cvt.rmi.u32: below 0 the
    cell is 0 and fr = pos < 0, so the weights leave [0, 1]), fr = pos - g."""
    f32 = np.float32
    res, mr = lay.resolutions[level], lay.max_res
    pos = np.asarray(x, f32) * f32(res - 1) + f32(0.5)                                   # triplane.py:56
    g = np.floor(np.maximum(pos, f32(0))).astype(np.uint32)                              # :57
    fr = pos - g.astype(f32)                                                             # :58
    a = [(f32(1) - fr[:, k], fr[:, k]) for k in range(3)]                                # :67, :70
    q = [tuple((g[:, k] + np.uint32(b)).astype(f32) / f32(res) * f32(mr - 1) for b in (0, 1))
         for k in range(3)]                                                              # :73-76
    return a, q


def triplane_ori(q, mr, clamp=True):
    """u32(q), truncated, clipped to max_res-1 when `clamp` (the kernel's one deviation from the reference)."""
    o = q.astype(np.uint32)
    return np.minimum(o, np.uint32(mr - 1)) if clamp else o


def corner_entry(lay, ori, fd, c):
    """Float index of feature 0 of corner c of plane fd: bit 0 picks the first axis' g+1, bit 1 the second's
    (triplane.py:60-87).  ori[k][b]: the max_res-grid coordinate of axis k, corner bit b."""
    d0, d1 = PLANES[fd]
    mr = lay.max_res
    index = ori[d0][c & 1].astype(np.int64) + ori[d1][c >> 1].astype(np.int64) * mr
    return (fd * mr * mr + index) * lay.feat_dim


def corner_weight(a, fd, c):
    d0, d1 = PLANES[fd]
    return a[d0][c & 1] * a[d1][c >> 1]          # ((1 * a_d0) * a_d1) in fp32, triplane.py:61-70


def triplane_numpy(xyz, table, lay, acc=np.float32, clamp=False):
    """Vectorised restatement of triplane_encoder_kernel (triplane.py:35-98): the geometry in fp32 exactly as the
    kernel computes it, the feature arithmetic in ``acc`` (fp32: bit-exact; fp64: for finite differences).
    clamp: the max_res-grid coordinate clipped to [0, max_res-1] as the kernel clips it (positions outside [0, 1]).
    `table`: an array or a callable of the float index.  Returns [n, L*F] with column j*L + level."""
    x = np.asarray(xyz, np.float32)
    n, L, F, mr = x.shape[0], lay.levels, lay.feat_dim, lay.max_res
    at = table if callable(table) else _table_at(np.asarray(table).astype(acc, copy=False))
    out = np.zeros((n, L * F), acc)
    cols = np.arange(F)
    for level in range(L):
        a, q = triplane_axes(x, lay, level)
        ori = [[triplane_ori(qb, mr, clamp) for qb in qk] for qk in q]
        lf = np.zeros((3, n, F), acc)
        for fd in range(3):
            for c in range(4):
                w = corner_weight(a, fd, c).astype(acc)
                t = np.asarray(at(corner_entry(lay, ori, fd, c)[:, None] + cols)).astype(acc, copy=False)
                lf[fd] = lf[fd] + w[:, None] * t                                         # :90-92
        for j in range(F):
            cp = np.ones(n, acc)
            for fd in range(3):
                cp = cp * lf[fd, :, j]                                                   # :94-96
            out[:, j * L + level] = cp
    return out


def _scatter(keys, vals, mags, cnts):
    """Sum rows of vals / mags [m, F] and cnts [m] by key: (unique keys, sums [u, F], sums [u, F], counts [u])."""
    uq, inv = np.unique(keys, return_inverse=True)
    F = vals.shape[1]
    ref = np.stack([np.bincount(inv, vals[:, j], uq.size) for j in range(F)], 1)
    mag = np.stack([np.bincount(inv, mags[:, j], uq.size) for j in range(F)], 1)
    return uq, ref, mag, np.bincount(inv, cnts, uq.size)


def np_triplane_bwd_f64(xn, table_at, dout, lay):
    """fp64 reference of the table backward (triplane_bwd_kernel): the geometry and the corner weights w in fp32
    exactly as the kernel computes them; after that everything in fp64: lf[fd][j] = sum_c w_c t[e_c + j] and, per
    (plane fd, corner c, column j), term = w_c * dy_j * prod_{fd' != fd} lf[fd'][j] added to t's float e_c + j.
    Rows whose dy is zero in all F columns of a level are skipped, as the kernel skips them.

    Returns (idx, ref, mag, cnt) over the floats some term reaches, idx sorted: ref the sum of the terms, mag the sum of
    |w_c dy_j| * prod_{fd' != fd} M[fd'][j] with M[fd'][j] = sum_c |w_c t| (>= |lf|, the scale of every rounding in
    the term), cnt the number of terms (contributions of corners that land on the same entry count once each)."""
    x = np.asarray(xn, np.float32)
    n, L, F, mr = x.shape[0], lay.levels, lay.feat_dim, lay.max_res
    dy_all = np.asarray(dout, np.float32).reshape(n, F, L).astype(np.float64)    # column j*L + level
    cols = np.arange(F)
    parts = []
    for level in range(L):
        dy = dy_all[:, :, level]
        live = (dy != 0).any(1)
        xl, dy = x[live], dy[live]
        if xl.shape[0] == 0:
            continue
        a, q = triplane_axes(xl, lay, level)
        ori = [[triplane_ori(qb, mr) for qb in qk] for qk in q]
        e = [[corner_entry(lay, ori, fd, c) for c in range(4)] for fd in range(3)]
        w = [[corner_weight(a, fd, c).astype(np.float64) for c in range(4)] for fd in range(3)]
        lf, M = np.zeros((3, xl.shape[0], F)), np.zeros((3, xl.shape[0], F))
        for fd in range(3):
            for c in range(4):
                wt = w[fd][c][:, None] * np.asarray(table_at(e[fd][c][:, None] + cols), np.float64)
                lf[fd] += wt
                M[fd] += np.abs(wt)
        keys, vals, mags = [], [], []
        for fd in range(3):
            o1, o2 = [k for k in range(3) if k != fd]
            p, pm = dy * lf[o1] * lf[o2], np.abs(dy) * M[o1] * M[o2]
            for c in range(4):
                keys.append(e[fd][c])
                vals.append(w[fd][c][:, None] * p)
                mags.append(np.abs(w[fd][c])[:, None] * pm)
        keys = np.concatenate(keys)
        parts.append(_scatter(keys, np.concatenate(vals), np.concatenate(mags), np.ones(keys.size)))
    if not parts:
        return (np.zeros(0, np.int64), np.zeros(0), np.zeros(0), np.zeros(0, np.int64))
    uq, ref, mag, cnt = _scatter(*(np.concatenate(p) for p in zip(*parts)))
    idx = (uq[:, None] + cols).reshape(-1)
    return idx, ref.reshape(-1), mag.reshape(-1), np.repeat(np.rint(cnt).astype(np.int64), F)


def _check_triplane_scatter(got, prefill, idx, ref, mag, cnt, what):
    """got, prefill: fp32 gradient after and before the backward; (idx, ref, mag, cnt) of np_triplane_bwd_f64.
    Every float in idx within gamma(k + C) * (|prefill| + mag) of prefill + ref, every other float bit-unchanged, and
    a non-finite float fails.  Returns the largest err / bound.

    The bound, gamma(m) = m u / (1 - m u), u = 2^-24, k = cnt, C = C_TERM = 11 (Higham, Accuracy and Stability of
    Numerical Algorithms, ch. 3; the kernel forms one term in fp32 as lf sums, two products, one product by w):
      - lf = ((0 + w0 t0) + w1 t1) + w2 t2) + w3 t3: four products and three adds (0 + x is exact), so
        |lf^ - lf| <= gamma(4) M, and |lf_a^ lf_b^ - lf_a lf_b| <= ((1 + gamma(4))^2 - 1) M_a M_b <= gamma(8) M_a M_b;
      - dlf = (dy * lf_a^) * lf_b^ (or dy * (lf_a^ * lf_b^)): two products; w * dlf: one more.  So the term is
        w dy lf_a lf_b + E with |E| <= gamma(8 + 3) |w dy| M_a M_b: 11 roundings;
      - k atomic adds onto prefill, in any order, are a recursive sum of k + 1 numbers: each term and prefill is
        carried through at most k roundings, so the total error is <= gamma(k) |prefill| + sum (gamma(k) + gamma(11)
        (1 + gamma(k))) mag_term <= gamma(k + 11) (|prefill| + mag).
    The fp32 oracle (oracle/triplane.c) forms the same products and sums sequentially, so the bound holds for it too.
    The geometry (w and the entries) is computed by the reference exactly as the kernel computes it, so it carries no
    error term; no term is subnormal for the inputs of these tests."""
    got = np.asarray(got, np.float32)
    prefill = np.asarray(prefill, np.float32)
    assert got.shape == prefill.shape, what
    rest = np.ones(got.size, bool)
    rest[idx] = False
    changed = np.flatnonzero(rest & (got.view(np.uint32) != prefill.view(np.uint32)))
    assert changed.size == 0, f"{what}: {changed.size} floats no term reaches were written, e.g. float {changed[0]}"
    g, p = got[idx].astype(np.float64), prefill[idx].astype(np.float64)
    assert np.isfinite(p).all() and np.isfinite(ref).all() and np.isfinite(mag).all(), what
    err = np.abs(g - (p + ref))
    m = (cnt + C_TERM) * U
    bound = m / (1 - m) * (np.abs(p) + mag)
    bad = np.flatnonzero(~(err <= bound))     # a NaN or inf float fails too
    assert bad.size == 0, (f"{what}: {bad.size} of {idx.size} floats outside the bound, e.g. float {idx[bad[0]]}: err "
                           f"{err[bad[0]]:.3e} bound {bound[bad[0]]:.3e} k {cnt[bad[0]]} ref {ref[bad[0]]:.6e}")
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(bound > 0, err / bound, 0.0)
    return float(ratio.max()) if ratio.size else 0.0
