"""fp64 restatement of the fused head with depth supervision (ngp_ray_head_fused_depth, DESIGN.md §6h) and its
comparator (tests/test_depth.py on the CPU, tests/test_gpu_depth.py on the GPU).

loss_sum = sum_r |out_r - gt_r|^2 + 3 w_d sum_r loss_ray_r + 3 w_z sum_r v_r (D_r - D^_r)^2, with D_r = sum_k w_k t_k,
v_r = 1 where D^_r is finite and > 0; dL/dD_r = scale 2 w_z v_r (D_r - D^_r) / n_rays enters the compositing's
transpose as its g_depth does.  The background is a constant (bg a float) or per-ray colours (bg = (colours, alpha or
None, b_load)), as in ngp_ray_head_fused_random_bg.
"""
import numpy as np

from composite_ref import U, _check_composite_bwd, kernel_termination, np_composite_f64, termination_window
from test_gpu_graph_step_distortion import np_distortion_f64


def depth_valid(depth_gt):
    d = np.asarray(depth_gt, np.float64)
    with np.errstate(invalid='ignore'):
        return np.isfinite(d) & (d > 0)


def head_ref_depth(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, w_z, depth_gt, thr, n_active=None, faults=()):
    """fp64 head.  Faults (comparator tests): "no_gz" (the depth gradient does not reach the compositing), "coef_valid"
    (normalised by the number of rays with a target instead of n_rays), "invalid_as_zero" (rays without a target are
    pulled towards depth 0) and "bg_in_depth" (the depth gets a background term (1 - opacity) t_far)."""
    n, S = rays_a.shape[0], sig.size
    z, zs = np.zeros(n), np.zeros(S)
    fwd = np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, z, z, np.zeros((n, 3)), zs, n_active=n_active)
    if isinstance(bg, tuple):
        cols, alpha, b_load = bg
        c = cols.astype(np.float64)
        tgt = gt.astype(np.float64)
        if alpha is not None:
            tgt = tgt + (c - b_load) * (1 - alpha.astype(np.float64))[:, None]
    else:
        c = np.full((n, 3), float(bg))
        tgt = gt.astype(np.float64)
    out = fwd["rgb"] + c * (1 - fwd["op"])[:, None]
    dd = out - tgt
    g = scale * 2 * dd / (3 * n)
    go = -(c * g).sum(1)
    loss_ray, lmag, dw, gmag = np_distortion_f64(fwd["w"], deltas, ts, rays_a)
    gw = scale * w_d / n * dw
    # the depth term
    v = depth_valid(depth_gt)
    if "invalid_as_zero" in faults:
        v = np.ones(n, bool)
    dh = np.where(depth_valid(depth_gt), np.asarray(depth_gt, np.float64), 0.0)
    D = fwd["dep"].copy()
    if "bg_in_depth" in faults:
        for r, s0, cnt in rays_a:
            if cnt:
                D[r] += (1 - fwd["op"][r]) * float(ts[s0 + cnt - 1])
    dz = np.where(v, D - dh, 0.0)
    n_z = max(int(v.sum()), 1) if "coef_valid" in faults else n
    gz = np.zeros(n) if "no_gz" in faults else scale * 2 * w_z * dz / n_z
    ref = np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, gz, g, gw, n_active=n_active)
    # tolerance scale: |dL/dw| replaced by its sum of |terms|, |dL/dD| by scale 2 w_z v (D + D^) / n (D carries the
    # compositing's relative error, which (D - D^) does not shrink)
    gz_mag = scale * 2 * w_z * np.where(v, D + dh, 0.0) / n
    ref["mag"] = np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, gz_mag, g, scale * w_d / n * gmag,
                                  n_active=n_active)["mag"]
    loss = (dd ** 2).sum() + 3 * w_d * loss_ray.sum() + 3 * w_z * (dz ** 2).sum()
    return dict(fwd=fwd, out=out, dd=dd, ref=ref, loss=loss, loss_ray=loss_ray, lmag=lmag, D=D, dz=dz, v=v, gz=gz)


def check_head_depth(got, sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, w_z, depth_gt, thr, half, what,
                     faults=()):
    """Comparator of one head launch, got = (loss_sum, opacity, rgb, dsig, drgbs) as numpy: the bounds of
    tests/test_gpu_graph_step_distortion.py::check_head_dist, plus the depth term's.  D is a sum of w_k t_k with w_k
    off by a few k u of itself (k = N + 4 / min a), so |D - D_exact| <= 8 k u D; the per-ray term v (D - D^)^2 is then
    off by 2 |D - D^| 8 k u D + 8 u (D - D^)^2.  Returns the reference and the largest measured errors."""
    ls, op, rgb, dsig, drgbs = got
    n_lo, n_hi, n64 = termination_window(sig, deltas, rays_a, thr)
    n_k = kernel_termination(dsig, drgbs, rays_a)
    bad = np.flatnonzero((n_k < n_lo) | (n_k > n_hi))
    assert bad.size == 0, f"{what}: {bad.size} rays stop outside the fp32 window of the threshold"
    h = head_ref_depth(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, w_z, depth_gt, thr, n_active=n_k,
                       faults=faults)
    fwd, out, dd, ref = h["fwd"], h["out"], h["dd"], h["ref"]
    _check_composite_bwd(dsig, drgbs, ref, half, what)
    k = fwd["kray"]
    assert (np.abs(op - fwd["op"]) <= 8 * k * U * fwd["op"] + 1e-30).all(), f"{what}: opacity"
    e_out = 8 * k[:, None] * U * (np.abs(out) + 2)
    assert (np.abs(rgb - out) <= e_out).all(), f"{what}: rgb"
    e_z = 3 * w_z * (2 * np.abs(h["dz"]) * 8 * k * U * np.abs(h["D"]) + 8 * U * h["dz"] ** 2)
    tol = ((2 * np.abs(dd) * e_out).sum() + 3 * w_d * (8 * k * U * h["lmag"]).sum() + e_z.sum()
           + 16 * rays_a.shape[0] * U * ((dd ** 2).sum() + 3 * w_d * h["lmag"].sum() + 3 * w_z * (h["dz"] ** 2).sum()))
    err_loss = abs(float(np.ravel(ls)[0]) - h["loss"])
    assert err_loss <= tol, f"{what}: loss_sum {np.ravel(ls)[0]} vs {h['loss']} (tol {tol:.3e})"
    act = ref["active"]
    rel = np.abs(dsig.astype(np.float64) - ref["dsig"])[act] / np.maximum(8 * ref["k"] * U * ref["mag"], 1e-300)[act]
    return h, dict(loss_err=err_loss, loss_tol=tol, dsig_err_over_tol=float(rel.max()) if rel.size else 0.0)
