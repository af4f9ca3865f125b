"""SSIM in fp64, written from its definition (DESIGN.md §6e; torchmetrics' StructuralSimilarityIndexMeasure with
data_range=1, Gaussian window sigma 1.5 over 11 taps, k1 = 0.01, k2 = 0.03), with the per-image error bound that
ngp_ssim is judged by and a numpy fp32 copy of the kernel's arithmetic into which mistakes can be planted.

Images are fp32 [H*W, 3] (or [B, H*W, 3]), H rows of W pixels, RGB interleaved.  For each channel and each of the
(H-10) x (W-10) positions where the 11 x 11 window g x g lies inside the image, the window-weighted moments mu_x,
mu_y, E[x^2], E[y^2], E[xy] give
    s = (2 mu_x mu_y + C1)(2 sigma_xy + C2) / ((mu_x^2 + mu_y^2 + C1)(sigma_x^2 + sigma_y^2 + C2)),
sigma_x^2 = E[x^2] - mu_x^2, sigma_y^2 = E[y^2] - mu_y^2, sigma_xy = E[xy] - mu_x mu_y, C1 = 0.01^2, C2 = 0.03^2.
The SSIM of an image is the mean of s over the 3 channels and the valid positions.
"""
import numpy as np

R = 5
TAPS = 2 * R + 1
SIGMA = 1.5
C1, C2 = 0.01 ** 2, 0.03 ** 2
U = 2.0 ** -24                       # fp32 unit roundoff
# the kernel's tiling (csrc/metrics.cu), which sets the length of its summation chains
KERNEL_TX, KERNEL_SUM_THREADS = 96, 256
SLACK = 1.1                          # covers what bound() drops: gamma_n = n u / (1 - n u) vs n u, and products of
                                     # the two passes' relative errors (each below 1e-5)

FAULTS = ("taps10", "full", "c_swap", "channel_stride")


def window(taps=TAPS):
    """g[i] = exp(-(i/1.5)^2 / 2) / sum, i = -5 ... taps - 6 (taps = 11: the symmetric window), fp64."""
    i = np.arange(taps, dtype=np.float64) - R
    e = np.exp(-0.5 * (i / SIGMA) ** 2)
    return e / e.sum()


def images(a, H, W):
    """[H*W, 3] or [B, H*W, 3] -> fp64 [B, 3, H, W] (channel planes of the interleaved rows)."""
    a = np.asarray(a)
    a = a.reshape(-1, H * W, 3)
    return a.reshape(-1, H, W, 3).transpose(0, 3, 1, 2).astype(np.float64)


def filt(f, g):
    """Valid-position separable filter: horizontal sum over the columns, then vertical over the rows, explicitly."""
    T = len(g)
    Wo, Ho = f.shape[-1] - T + 1, f.shape[-2] - T + 1
    h = sum(g[k] * f[..., :, k:k + Wo] for k in range(T))
    return sum(g[k] * h[..., k:k + Ho, :] for k in range(T))


def moments(x, y, g=None):
    g = window() if g is None else g
    return filt(x, g), filt(y, g), filt(x * x, g), filt(y * y, g), filt(x * y, g)


def ssim_map(mx, my, exx, eyy, exy, c1=C1, c2=C2):
    vx, vy, cxy = exx - mx * mx, eyy - my * my, exy - mx * my
    return (2 * mx * my + c1) * (2 * cxy + c2) / ((mx * mx + my * my + c1) * (vx + vy + c2))


def ssim(pred, target, H, W):
    """fp64 SSIM per image -> [B]."""
    x, y = images(pred, H, W), images(target, H, W)
    return ssim_map(*moments(x, y)).mean(axis=(1, 2, 3))


def bound(pred, target, H, W):
    """Per-image bound on |ngp_ssim - ssim| -> [B].

    Moments.  The kernel forms each moment m = sum_ij g_i g_j f_ij (f = x, y, x^2, y^2, xy) as a horizontal pass of 11
    fp32 products and adds per input row, then a vertical pass of 11 more.  The fp32 weights are within u of g, every
    product and add rounds once, and each chain has 10 adds, so |dm| <= (1 + 2 + 10 + 1 + 1 + 10) u m_abs, 25 u m_abs
    with m_abs = sum_ij g_i g_j |f_ij| (taken as 26 u m_abs).
    Formula.  Each step's error is propagated exactly to first order, from the fp64 values:
      d(mu^2) <= (2|mu| + dmu) dmu + u mu^2,   d(sigma^2) = d(E[x^2] - mu^2) <= dE + d(mu^2) + u (E + mu^2 + dE + d(mu^2))
    (the cancellation: the subtraction's inputs carry errors relative to E[x^2] ~ mu^2, not to the small sigma^2), and
    the same for sigma_xy; the four factors A1 = 2 mu_x mu_y + C1, A2 = 2 sigma_xy + C2, B1 = mu_x^2 + mu_y^2 + C1,
    B2 = sigma_x^2 + sigma_y^2 + C2 add the rounding of the fp32 constant and of each add; N = A1 A2, D = B1 B2 and
      |s~ - s| <= (dN D + |N| dD) / (D (D - dD)) + u (|N| + dN) / (D - dD).
    The floors: B1 >= C1 and B2 >= C2 exactly (sigma^2 >= 0 for a window of weight 1), so D - dD stays positive unless
    dD itself reaches C1 C2; then the bound is infinite.
    Mean.  Every s reaches its image's sum through at most L = 3 ceil(Wo/96) + 5 + 2 + ceil(Ho/256) + 8 adds (the row
    accumulator over channels and x-tiles, the warp tree, the 3 warps, the per-thread row sum, the 256-thread tree), so
    the mean is off by at most mean |ds| + (L + 1) u mean |s|.  The result is that times SLACK.
    The bound adds worst cases; in practice rounding errors of neighbouring positions cancel, so measured errors sit far
    below it, yet the planted mistakes of kernel_np exceed it (tests/test_ssim.py)."""
    x, y = images(pred, H, W), images(target, H, W)
    g = window()
    mx, my, exx, eyy, exy = moments(x, y, g)
    ax, ay, axy = filt(np.abs(x), g), filt(np.abs(y), g), filt(np.abs(x * y), g)
    cm = 26 * U
    dmx, dmy, dexx, deyy, dexy = cm * ax, cm * ay, cm * exx, cm * eyy, cm * axy

    def dsq(m, dm):
        return (2 * np.abs(m) + dm) * dm + U * m * m

    def dsub(e, de, p, dp):
        return de + dp + U * (np.abs(e) + np.abs(p) + de + dp)

    mxx, myy, mxy = mx * mx, my * my, mx * my
    dmxx, dmyy = dsq(mx, dmx), dsq(my, dmy)
    dmxy = np.abs(mx) * dmy + np.abs(my) * dmx + dmx * dmy + U * np.abs(mxy)
    vx, vy, cxy = exx - mxx, eyy - myy, exy - mxy
    dvx, dvy, dcxy = dsub(exx, dexx, mxx, dmxx), dsub(eyy, deyy, myy, dmyy), dsub(exy, dexy, mxy, dmxy)
    A1, A2 = 2 * mxy + C1, 2 * cxy + C2
    B1, B2 = mxx + myy + C1, vx + vy + C2
    dA1 = 2 * dmxy + U * (np.abs(A1) + 2 * dmxy + C1)
    dA2 = 2 * dcxy + U * (np.abs(A2) + 2 * dcxy + C2)
    dB1 = dmxx + dmyy + U * (2 * (B1 + dmxx + dmyy) + C1)
    dB2 = dvx + dvy + U * (2 * (np.abs(vx) + np.abs(vy) + dvx + dvy + C2) + C2)

    def dprod(a, da, b, db):
        return np.abs(a) * db + np.abs(b) * da + da * db + U * (np.abs(a) + da) * (np.abs(b) + db)

    N, D = A1 * A2, B1 * B2
    dN, dD = dprod(A1, dA1, A2, dA2), dprod(B1, dB1, B2, dB2)
    lo = D - dD
    with np.errstate(divide="ignore", invalid="ignore"):
        ds = np.where(lo > 0, (dN * D + np.abs(N) * dD) / (D * lo) + U * (np.abs(N) + dN) / lo, np.inf)
    s = N / D
    Ho, Wo = H - 2 * R, W - 2 * R
    L = 3 * -(-Wo // KERNEL_TX) + 5 + 2 + -(-Ho // KERNEL_SUM_THREADS) + 8
    mean_abs = np.abs(s).mean(axis=(1, 2, 3))
    return SLACK * (ds.mean(axis=(1, 2, 3)) + (L + 1) * U * mean_abs)


def check(got, pred, target, H, W, what=""):
    """Assert that every image's result lies within bound() of the fp64 SSIM; returns the largest error/bound."""
    got = np.asarray(got, dtype=np.float64).reshape(-1)
    ref, b = ssim(pred, target, H, W), bound(pred, target, H, W)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = np.abs(got - ref)
    bad = ~(err <= b)
    assert not bad.any(), (f"{what}: images {np.nonzero(bad)[0].tolist()} off the fp64 bound: got {got[bad]}, "
                           f"fp64 {ref[bad]}, err {err[bad]}, bound {b[bad]}")
    return float((err / b).max())


# ---- a numpy fp32 copy of the kernel's arithmetic, for fault injection -------------------------------------------
def kernel_np(pred, target, H, W, fault=None):
    """fp32 SSIM per image computed the kernel's way: fp32 weights, a horizontal 11-tap pass of the five moments per
    input row, the vertical pass in tap order, the formula in fp32, fp32 sums.  ``fault`` plants one mistake:
      taps10          a 10-tap window (i = -5 ... 4, renormalised)
      full            the same-size map: reflect-pad by 5 and average over all H x W positions
      c_swap          C1 and C2 swapped
      channel_stride  the channels read as if the image were planar [3, H, W]"""
    f32 = np.float32
    g = window(10 if fault == "taps10" else TAPS).astype(f32)
    c1, c2 = (f32(C2), f32(C1)) if fault == "c_swap" else (f32(C1), f32(C2))
    p = np.asarray(pred, dtype=f32).reshape(-1, H * W * 3)
    t = np.asarray(target, dtype=f32).reshape(-1, H * W * 3)
    out = []
    for a, b in zip(p, t):
        if fault == "channel_stride":
            x, y = a.reshape(3, H, W), b.reshape(3, H, W)
        else:
            x, y = a.reshape(H, W, 3).transpose(2, 0, 1), b.reshape(H, W, 3).transpose(2, 0, 1)
        if fault == "full":
            pad = ((0, 0), (R, R), (R, R))
            x, y = np.pad(x, pad, mode="reflect"), np.pad(y, pad, mode="reflect")
        T = len(g)
        Wo, Ho = x.shape[-1] - T + 1, x.shape[-2] - T + 1
        h = [np.zeros((3, x.shape[1], Wo), f32) for _ in range(5)]
        for k in range(T):
            xs, ys = x[:, :, k:k + Wo], y[:, :, k:k + Wo]
            gx, gy = g[k] * xs, g[k] * ys
            h[0] += gx
            h[1] += gy
            h[2] += gx * xs
            h[3] += gy * ys
            h[4] += gx * ys
        m = [np.zeros((3, Ho, Wo), f32) for _ in range(5)]
        for k in range(T):
            for i in range(5):
                m[i] += g[k] * h[i][:, k:k + Ho, :]
        mx, my, exx, eyy, exy = m
        mxx, myy, mxy = mx * mx, my * my, mx * my
        s = ((f32(2) * mxy + c1) * (f32(2) * (exy - mxy) + c2)) / ((mxx + myy + c1) * ((exx - mxx) + (eyy - myy) + c2))
        out.append(f32(s.sum(axis=(0, 2), dtype=f32).sum(dtype=f32) / f32(s.size)))
    return np.array(out, dtype=f32)
