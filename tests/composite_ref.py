"""fp64 references for the volume compositing and its backward (tests/test_gpu_step_kernels.py,
tests/test_gpu_graph_step_grads.py).

- `np_composite_f64`: the compositing (volume_train.py:22-48) and its transpose, per ray, with the per-sample error
  scale `_check_composite_bwd` holds a kernel's dL/dsigma and dL/drgb to.
- `termination_window`: where an fp32 kernel may legitimately stop a ray.  A kernel stops at the first sample whose
  fp32 transmittance is not above the threshold; when the exact transmittance lies within the fp32 error of the
  threshold, either choice is correct.  `kernel_termination` reads the choice a kernel made from its gradients, so
  that the fp64 reference can be built with the same termination index instead of being judged against the other.
"""
import numpy as np

U = 2.0 ** -24          # fp32 unit roundoff


def np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, gd, gr, gw, n_active=None):
    """fp64 restatement of the compositing (volume_train.py:22-48) and its transpose, per ray: w_s = a_s T_s while
    T_s > thr.  Returns forward sums, dsigma, drgb and, for the tolerances, the sum of |terms| of every dsigma and the
    conditioning factor N + 4 / min a of every ray (a = 1 - exp(-sigma delta) carries an absolute fp32 error).
    `n_active[ray]`, when given, is the number of samples the ray composites (a termination index chosen inside the
    fp32 error window, see kernel_termination); without it no sample may lie near the threshold."""
    S, n = sig.size, rays_a.shape[0]
    out = dict(op=np.zeros(n), rgb=np.zeros((n, 3)), dep=np.zeros(n), dsig=np.zeros(S), drgb=np.zeros((S, 3)),
               mag=np.zeros(S), w=np.zeros(S), k=np.zeros(S), kray=np.ones(n), active=np.zeros(S, bool))
    c_all = rgbs.astype(np.float64)
    for r, s0, cnt in rays_a:
        if cnt == 0:
            continue
        sl = slice(s0, s0 + cnt)
        x = sig[sl].astype(np.float64) * deltas[sl].astype(np.float64)
        a = -np.expm1(-x)
        Tn = np.exp(-np.cumsum(x))                   # T after each sample
        Tb = np.concatenate([[1.0], Tn[:-1]])        # T before
        if n_active is None:
            act = Tb > thr
            assert np.all(np.abs(np.log(Tb / thr)) > 1e-2), "a sample too close to the threshold for an fp64 reference"
        else:
            act = np.arange(cnt) < n_active[r]
        w = np.where(act, a * Tb, 0.0)
        c, t = c_all[sl], ts[sl].astype(np.float64)
        G = c @ gr[r].astype(np.float64) + gd[r] * t + go[r] + gw[sl]
        Gabs = np.abs(c) @ np.abs(gr[r]).astype(np.float64) + abs(gd[r]) * np.abs(t) + abs(go[r]) + np.abs(gw[sl])
        later = np.concatenate([np.cumsum((w * G)[::-1])[::-1][1:], [0.0]])
        later_abs = np.concatenate([np.cumsum((w * Gabs)[::-1])[::-1][1:], [0.0]])
        d = deltas[sl].astype(np.float64)
        out["dsig"][sl] = np.where(act, d * (Tn * G - later), 0.0)
        # T_{s+1} = T_s (1 - a_s) is off by ~u T_s, not u T_{s+1}, where a_s rounds to 1 in fp32
        out["mag"][sl] = d * (Tb * Gabs + later_abs)
        out["drgb"][sl] = w[:, None] * gr[r].astype(np.float64)[None, :]
        out["w"][sl], out["active"][sl] = w, act
        out["op"][r], out["rgb"][r], out["dep"][r] = w.sum(), w @ c, w @ t
        out["kray"][r] = cnt + 4.0 / a[act].min()
        out["k"][sl] = out["kray"][r]
    return out


def _check_composite_bwd(dsig, drgbs, ref, half, what):
    act = ref["active"]
    assert not dsig[~act].any() and not drgbs[~act].any(), f"{what}: gradient of a sample after termination"
    err = np.abs(dsig.astype(np.float64) - ref["dsig"])
    tol = 8 * ref["k"] * U * ref["mag"]
    bad = np.flatnonzero(err > tol)
    assert bad.size == 0, f"{what}: dsigma of {bad.size} samples, first {bad[0]}: err {err[bad[0]]:.3e} tol {tol[bad[0]]:.3e}"
    d = drgbs.astype(np.float64)
    tol = 8 * ref["k"][:, None] * U * np.abs(ref["drgb"]) + (2.0 ** -11 * np.abs(ref["drgb"]) + 2.0 ** -24 if half else 0)
    assert (np.abs(d - ref["drgb"]) <= tol).all(), f"{what}: drgb"


def termination_window(sig, deltas, rays_a, thr):
    """Per ray (indexed by ray id): (n_lo, n_hi, n64).  An fp32 kernel's transmittance before sample s is bracketed by
    an interval of the exact one: each factor 1 - a_j = exp(-x_j) (x_j = sigma_j delta_j) is off by
    e_j (x_j + 3) u + 2u absolutely (the product x_j, expf, then 1 - a in fp32) and every product it takes part in
    (the warp scan and the chunk carry) rounds by at most 8 u.  Samples whose bracket lies above fp32(thr) are active
    in any correct kernel (the first n_lo), those whose bracket lies at or below it are not (from n_hi on).
    n64 is the fp64 decision."""
    thr32 = float(np.float32(thr))
    n = rays_a.shape[0]
    n_lo, n_hi, n64 = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64)
    for r, s0, cnt in rays_a:
        if cnt == 0:
            continue
        x = sig[s0:s0 + cnt].astype(np.float64) * deltas[s0:s0 + cnt].astype(np.float64)
        e = np.exp(-x)
        lo = np.maximum(e * (1 - (x + 3) * U) - 2 * U, 0.0) * (1 - 8 * U)
        hi = np.minimum((e * (1 + (x + 3) * U) + 2 * U) * (1 + 8 * U), 1.0 + 16 * U)
        T_lo = np.concatenate([[1.0], np.cumprod(lo)[:-1]])
        T_hi = np.concatenate([[1.0], np.cumprod(hi)[:-1]])
        Tb = np.concatenate([[1.0], np.exp(-np.cumsum(x))[:-1]])
        # leading runs: the transmittance only falls, so each decision is a prefix
        n_lo[r] = int(np.argmin(T_lo > thr32)) if not (T_lo > thr32).all() else cnt
        n_hi[r] = int(np.argmin(T_hi > thr32)) if not (T_hi > thr32).all() else cnt
        n64[r] = int(np.argmin(Tb > thr)) if not (Tb > thr).all() else cnt
    return n_lo, n_hi, n64


def kernel_termination(dsig, drgbs, rays_a):
    """Per ray: the number of samples a kernel composited, read as one past the last sample with a non-zero
    dL/dsigma or dL/drgb (the kernel writes 0 to every sample after the ray's termination)."""
    nz = (np.asarray(dsig) != 0) | (np.asarray(drgbs) != 0).any(1)
    n_k = np.zeros(rays_a.shape[0], np.int64)
    for r, s0, cnt in rays_a:
        idx = np.flatnonzero(nz[s0:s0 + cnt])
        n_k[r] = idx[-1] + 1 if idx.size else 0
    return n_k
