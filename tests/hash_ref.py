"""fp64 references and inputs for the hash-grid kernels (tests/test_gpu_hash_kernels.py, tests/test_gpu_step_kernels.py).

- `np_hash_bwd_f64`: the table backward as an fp64 scatter, with its per-entry error scale and contribution count;
  `_check_scatter` holds a kernel's gradient to it with a bound that is valid in any atomic order.
- `np_hash_dx_f64`: the input gradient dL/dx as the exact derivative of the forward, with its per-component error scale.
- Inputs: ray-coherent and world-space points, the AABB of NGP.density, and the device row counts (n_dev) of the
  graph-captured step, with the PAD rows every device-count test allocates past n_max.

The cell and the fractional position are computed in fp32 exactly as the forward does (tests/test_oracle.py
np_hash_encode), the fp16 kernels' cast of the grid coordinate (hash_encoder_half.py:132) included.
"""
import ctypes as C

import numpy as np

U = 2.0 ** -24          # fp32 unit roundoff
PAD = 1040              # > 1000: room for a kernel that ignored the clamp at n_dev = n_max + 1000


def n_dev_cases(n_max):
    """0, 1, a value below n_max, n_max, the capacity overflow of the graph step (reserved rows > capacity), and a
    negative count."""
    return sorted({0, 1, n_max // 2, n_max, n_max + 1000, -5})


def rows_of(n_dev, n_max):
    return min(n_max, max(n_dev, 0))


def _normalise(x, scale):
    """NGP.density's x = (x - xyz_min) / (xyz_max - xyz_min) in fp32, as oracle/train_step.py computes it."""
    lo, hi = np.float32(-scale), np.float32(scale)
    return ((x - lo) / (hi - lo)).astype(np.float32)


def _aabb6(scale):
    lo, hi = np.float32(-scale), np.float32(scale)
    return (C.c_float * 6)(lo, lo, lo, hi - lo, hi - lo, hi - lo)


def _world_points(rng, n, scale):
    """Uniform points of the box, the corners and face centres first, and one point in seven moved onto a face."""
    s = np.float32(scale)
    x = rng.uniform(-scale, scale, (n, 3)).astype(np.float32)
    special = np.array([[-s, -s, -s], [s, s, s], [s, -s, 0.25 * s], [-s, 0.1 * s, s], [0, s, -s], [s, 0, 0],
                        [-s, 0, 0], [0.5 * s, -0.5 * s, s]], np.float32)
    k = min(n, len(special))
    x[:k] = special[:k]
    idx = rng.choice(n, n // 7, replace=False) if n >= 7 else np.arange(0)
    x[idx, rng.integers(0, 3, idx.size)] = np.where(rng.random(idx.size) < 0.5, -s, s)
    return x


def _ray_points(rng, n, per_ray=100, step=0.0015):
    """Samples along rays in [0, 1]: consecutive rows share cells, as the march emits them (exercises the backward's
    register run-accumulation and its flushes)."""
    base = rng.random((n // per_ray + 1, 1, 3), dtype=np.float32) * 0.8 + 0.1
    d = rng.standard_normal((n // per_ray + 1, 1, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=2, keepdims=True)
    x = base + np.arange(per_ray, dtype=np.float32)[None, :, None] * step * d
    return x.reshape(-1, 3)[:n].clip(0, 1).astype(np.float32)


def grid_cell(xn, lay, lvl, half):
    """(g uint32 [n, 3], fractional position fp32 [n, 3]) of level `lvl`: pos = x * scale + 0.5 in fp32,
    g = floor(pos), frac = pos - g with g cast to fp16 first in the fp16 kernels.  Above 2048 an odd g rounds to an
    even neighbour there, so frac leaves [0, 1) and some trilinear weights are negative."""
    pos = (xn * np.float32(lay.scales[lvl])).astype(np.float32) + np.float32(0.5)
    g = np.floor(pos).astype(np.int64).astype(np.uint32)
    gf = g.astype(np.float16).astype(np.float32) if half else g.astype(np.float32)
    return g, pos - gf


def corner_entries(lay, lvl, g, c):
    """Table entry (level offset included) of corner c of cells g: under_hash on dense levels, fast_hash on hashed
    ones, then % map_size (hash_encoder.py:43-71)."""
    res = np.uint32(lay.resolutions[lvl])
    p = [g[:, d] + np.uint32((c >> d) & 1) for d in range(3)]
    if lvl < lay.begin_fast_hash_level:
        h = p[0] + p[1] * res + p[2] * (res * res)
    else:
        h = p[0] ^ (p[1] * np.uint32(2654435761)) ^ (p[2] * np.uint32(805459861))
    return lay.offsets[lvl] + (h % np.uint32(lay.map_sizes[lvl])).astype(np.int64)


def np_hash_bwd_f64(xn, dout, lay, half, levels):
    """fp64 reference of the table backward restricted to `levels`: the cell and the trilinear weights in fp32 exactly
    as np_hash_encode (tests/test_oracle.py), w * dy accumulated in fp64.  Returns (ref, sum of |w dy|, number of
    contributions) per table float.  Rows whose dy is all zero at a level are skipped (hash_encoder_half.py:210)."""
    n, F = xn.shape[0], lay.feat_dim
    dy_all = np.asarray(dout).reshape(n, lay.levels, F).astype(np.float64)
    E = lay.total_entries
    ref, mag, cnt = np.zeros((E, F)), np.zeros((E, F)), np.zeros(E, np.int64)
    with np.errstate(over="ignore"):
        for lvl in levels:
            dy = dy_all[:, lvl]
            live = (dy != 0).any(1)
            x, dy = xn[live], dy[live]
            g, frac = grid_cell(x, lay, lvl, half)
            for c in range(8):
                w = np.ones(x.shape[0], np.float32)
                for d in range(3):
                    w = w * (frac[:, d] if c & (1 << d) else np.float32(1) - frac[:, d])
                idx = corner_entries(lay, lvl, g, c)
                t = w.astype(np.float64)[:, None] * dy
                np.add.at(ref, idx, t)
                np.add.at(mag, idx, np.abs(t))
                np.add.at(cnt, idx, 1)
    return ref.reshape(-1), mag.reshape(-1), np.repeat(cnt, F)


def np_hash_dx_f64(xn, table, dout, lay, half):
    """fp64 reference of dL/dx = sum over levels and corners of scale * <table[corner], dy> * dw_c/dfrac: the
    derivative of the forward inside the cell of x, with the cell and fraction taken in fp32 exactly as the forward
    takes them (fp16 grid cast when `half`), and everything after that in fp64.  Returns (dx [n, 3], sum of |term|
    [n, 3]), where |term| = scale * sum_f |table * dy| * |w_a * w_b| (w_a, w_b: the weights of the two other axes),
    the scale of every rounding a kernel makes in the term and in its sum."""
    n, F = xn.shape[0], lay.feat_dim
    tab = np.asarray(table).reshape(-1, F).astype(np.float64)
    dy_all = np.asarray(dout).reshape(n, lay.levels, F).astype(np.float64)
    dx, mag = np.zeros((n, 3)), np.zeros((n, 3))
    with np.errstate(over="ignore"):
        for lvl in range(lay.levels):
            scale = float(np.float32(lay.scales[lvl]))
            g, frac = grid_cell(xn, lay, lvl, half)
            f = frac.astype(np.float64)
            a = [(1.0 - f[:, d], f[:, d]) for d in range(3)]       # a[d][bit]: the weight factor of axis d
            for c in range(8):
                prod = tab[corner_entries(lay, lvl, g, c)] * dy_all[:, lvl]
                v, v_abs = scale * prod.sum(1), scale * np.abs(prod).sum(1)
                for d in range(3):
                    e0, e1 = [e for e in range(3) if e != d]
                    wo = a[e0][(c >> e0) & 1] * a[e1][(c >> e1) & 1]
                    dx[:, d] += (v if c & (1 << d) else -v) * wo
                    mag[:, d] += v_abs * np.abs(wo)
    return dx, mag


def _level_ranges(lay):
    """Level ranges of the table backward.  "inner" drops the first and the last level: at L = 16 both its ends are
    odd, so the 16-byte staging of dL/dout (2 fp32 or 4 fp16 levels per load) must drop a column at either end."""
    L, fh = lay.levels, lay.begin_fast_hash_level
    mid = fh + (L - fh) // 2
    return {"all": (0, L), "dense": (0, fh), "hashed_coarse": (fh, mid), "hashed_fine": (mid, L),
            "last": (L - 1, L), "level3": (3, 4), "inner": (1, L - 1)}


def _level_slice(lay, a, b):
    F = lay.feat_dim
    return lay.offsets[a] * F, (lay.offsets[b] * F if b < lay.levels else lay.total_param_size)


def _check_scatter(got, prefill, ref, mag, cnt, lo, hi, what):
    """Inside [lo, hi): prefill + ref within (k + 4) u (|prefill| + sum |w dy|), untouched entries bit-unchanged.
    Outside: bit-unchanged.  The reference is finite, so a non-finite entry is outside the bound."""
    out = np.ones(got.size, bool)
    out[lo:hi] = False
    assert np.array_equal(got[out].view(np.uint32), prefill[out].view(np.uint32)), f"{what}: wrote outside its levels"
    g, p = got[lo:hi].astype(np.float64), prefill[lo:hi].astype(np.float64)
    r, m, k = ref[lo:hi], mag[lo:hi], cnt[lo:hi]
    untouched = k == 0
    assert np.array_equal(got[lo:hi][untouched].view(np.uint32), prefill[lo:hi][untouched].view(np.uint32)), \
        f"{what}: an entry no sample reaches was written"
    err = np.abs(g - (p + r))
    bound = (k + 4) * U * (np.abs(p) + m)
    bad = np.flatnonzero(~(err <= bound))     # a NaN or inf entry fails too
    assert np.isfinite(prefill[lo:hi]).all() and np.isfinite(r).all()
    assert bad.size == 0, (f"{what}: {bad.size} entries outside the bound, e.g. entry {lo + bad[0]}: err "
                           f"{err[bad[0]]:.3e} bound {bound[bad[0]]:.3e} k {k[bad[0]]} ref {r[bad[0]]:.6e}")
