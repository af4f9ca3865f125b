"""Integer restatement of the error map (DESIGN.md §6j, csrc/errmap.cu) in numpy: tile mapping, accumulate, rebuild,
sampling and weights.  Every quantity is an integer except the per-ray error (strict fp32, as numpy float32 computes
it) and the weight (fp64 products and quotient, rounded once to fp32)."""
import numpy as np

from oracle.oracle import philox4x32_10_np

FIX = 1 << 30
COUNTER_WORD = 0x656D0001


def tile_lo(k, length, R):
    return -(-np.asarray(k, np.int64) * length // R)   # ceil(k length / R)


def tile_pixels(geom):
    """n_t [T] int64."""
    n_img, W, H, R = geom
    k = np.arange(R + 1, dtype=np.int64)
    rows, cols = np.diff(tile_lo(k, H, R)), np.diff(tile_lo(k, W, R))
    return np.tile(np.outer(rows, cols).ravel(), n_img)


def tile_of(img, pix, geom):
    n_img, W, H, R = geom
    img = np.clip(np.asarray(img, np.int64), 0, n_img - 1)
    pix = np.clip(np.asarray(pix, np.int64), 0, W * H - 1)
    y, x = pix // W, pix % W
    return img * R * R + (y * R // H) * R + x * R // W


def errors_u(pred, target, bg_rgb=None, alpha=None, b_load=1.0):
    """u_r = floor(min(e_r, 3) 2^30) [n] uint64, e_r in strict fp32."""
    f = np.float32
    p, t = np.asarray(pred, f), np.asarray(target, f).copy()
    if bg_rgb is not None and alpha is not None:
        t = t + (np.asarray(bg_rgb, f) - f(b_load)) * (f(1) - np.asarray(alpha, f))[:, None]
    d = p - t
    e = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    with np.errstate(invalid="ignore"):
        e = np.where(e < f(3), e, f(3))
    return (e * f(FIX)).astype(np.uint64)


def accumulate(acc, cnt, pred, target, img, pix, geom, **kw):
    t = tile_of(img, pix, geom)
    np.add.at(acc, t, errors_u(pred, target, **kw).astype(np.int64))
    np.add.at(cnt, t, 1)


def limit(geom, p, q):
    n_img, W, H, R = geom
    N = n_img * W * H
    return ((q - p) * ((1 << 53) - N) - 1) // (N * q)


def rebuild(E, acc, cnt, geom, ema_shift=2, p=1, q=5):
    """(E', cdf, info) after one rebuild; acc and cnt are cleared in place."""
    E = np.asarray(E, np.int64).copy()
    seen = cnt > 0
    mean = np.where(seen, acc // np.maximum(cnt, 1), 0)
    E = np.where(seen, E + ((mean - E) >> ema_shift), E)
    acc[:] = 0
    cnt[:] = 0
    n_img, W, H, R = geom
    N = n_img * W * H
    lim = limit(geom, p, q)
    emax = int(E.max())
    k = 0
    while (emax >> k) > lim:
        k += 1
    n_t = tile_pixels(geom)
    Ep = E >> k
    S = int((n_t * Ep).sum())   # < 2^53 by the choice of k
    d = (q - p) * N
    c = max(1, (p * S + d - 1) // d)
    m = n_t * (Ep + c)
    cdf = np.cumsum(m)
    M = int(cdf[-1])
    assert M < (1 << 53) and M == S + c * N
    return E, cdf, {"k": k, "c": c, "S": S, "M": M, "emax": emax, "lim": lim}


def _mulhi64(x, M):
    """floor(x M / 2^64) for uint64 x and M < 2^53, exactly in uint64 pieces."""
    m32 = np.uint64(0xFFFFFFFF)
    s32 = np.uint64(32)
    xh, xl = x >> s32, x & m32
    mh, ml = np.uint64(M >> 32), np.uint64(M & 0xFFFFFFFF)
    lo = xl * ml
    t1 = xh * ml + (lo >> s32)
    t2 = xl * mh + (t1 & m32)
    return xh * mh + (t1 >> s32) + (t2 >> s32)


def sample(cdf, geom, seed, step, n):
    """(img [n], pix [n], w [n] fp32) of ngp_error_map_sample."""
    n_img, W, H, R = geom
    i = np.arange(n, dtype=np.uint64)
    r0, r1, r2, _ = philox4x32_10_np(i & np.uint64(0xFFFFFFFF), i >> np.uint64(32), np.uint32(step & 0xFFFFFFFF),
                                     np.uint32(COUNTER_WORD), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    cdf = np.asarray(cdf, np.int64)
    M = int(cdf[-1])
    x = (r0.astype(np.uint64) << np.uint64(32)) | r1.astype(np.uint64)
    v = _mulhi64(x, M).astype(np.int64)
    t = np.searchsorted(cdf, v, side="right")
    m_t = cdf[t] - np.where(t > 0, cdf[np.maximum(t - 1, 0)], 0)
    img, l = t // (R * R), t % (R * R)
    ty, tx = l // R, l % R
    y0, x0 = tile_lo(ty, H, R), tile_lo(tx, W, R)
    tw = tile_lo(tx + 1, W, R) - x0
    n_t = (tile_lo(ty + 1, H, R) - y0) * tw
    j = ((r2.astype(np.uint64) * n_t.astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
    pix = (y0 + j // tw) * W + x0 + j % tw
    N = float(n_img * W * H)
    w = ((np.float64(M) * n_t.astype(np.float64)) / (N * m_t.astype(np.float64))).astype(np.float32)
    return img, pix, w
