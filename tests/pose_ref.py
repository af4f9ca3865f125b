"""fp64 restatement of the camera extrinsics refinement (DESIGN.md §6i): Exp and the left Jacobian J_l of SO(3), the
corrected rays, and the pose gradient through torch.autograd."""
import numpy as np


def hat(w):
    w = np.asarray(w, np.float64)
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def so3_exp(w):
    """Rodrigues: I + sin(t)/t K + (1 - cos t)/t^2 K^2; the Taylor series below t = 1e-4."""
    w = np.asarray(w, np.float64)
    t = np.linalg.norm(w)
    K = hat(w)
    if t < 1e-4:
        A, B = 1 - t * t / 6, 0.5 - t * t / 24
    else:
        A, B = np.sin(t) / t, (1 - np.cos(t)) / (t * t)
    return np.eye(3) + A * K + B * K @ K


def so3_jl(w):
    """Left Jacobian: I + (1 - cos t)/t^2 K + (t - sin t)/t^3 K^2; the Taylor series below t = 1e-3."""
    w = np.asarray(w, np.float64)
    t = np.linalg.norm(w)
    K = hat(w)
    if t < 1e-3:
        B, C = 0.5 - t * t / 24, 1 / 6 - t * t / 120
    else:
        B, C = (1 - np.cos(t)) / (t * t), (t - np.sin(t)) / t ** 3
    return np.eye(3) + B * K + C * K @ K


def so3_log(R):
    """Rotation vector of a rotation matrix (angles below pi)."""
    c = np.clip((np.trace(R) - 1) / 2, -1.0, 1.0)
    t = np.arccos(c)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    if t < 1e-7:
        return v / 2
    return v * t / (2 * np.sin(t))


def rays_f64(dirs, img, poses, corr):
    """(rays_o, rays_d) fp64: d' = Exp(omega) R c, o' = o + tau; corr [n_img, 8]."""
    dirs, poses, corr = (np.asarray(a, np.float64) for a in (dirs, poses, corr))
    o = np.empty((len(dirs), 3))
    d = np.empty((len(dirs), 3))
    for i in range(len(dirs)):
        k = int(img[i])
        R = so3_exp(corr[k, 0:3]) @ poses[k, :, :3]
        d[i] = R @ dirs[i]
        o[i] = poses[k, :, 3] + corr[k, 4:7]
    return o, d


def pose_grad_autograd(dirs, img, poses, corr, ts, rays_a, dx):
    """dL/d(omega, tau) [n_img, 6] fp64 by torch.autograd through Rodrigues, for L = sum_s dx_s . x_s with
    x_s = o' + t_s d' of the ray owning row s (the colour network's direction held constant, as in §6i)."""
    import torch
    t64 = lambda a: torch.as_tensor(np.asarray(a, np.float64))  # noqa: E731
    n_img = poses.shape[0]
    w = t64(corr[:, 0:3]).clone().requires_grad_(True)
    tau = t64(corr[:, 4:7]).clone().requires_grad_(True)
    P = t64(poses)
    th = torch.sqrt((w * w).sum(1) + 1e-300)[:, None, None]
    z = torch.zeros(n_img, dtype=torch.float64)
    rows_k = [[z, -w[:, 2], w[:, 1]], [w[:, 2], z, -w[:, 0]], [-w[:, 1], w[:, 0], z]]
    K = torch.stack([torch.stack(r, -1) for r in rows_k], -2)
    small = (th < 1e-4)
    A = torch.where(small, 1 - th ** 2 / 6, torch.sin(th) / th)
    B = torch.where(small, 0.5 - th ** 2 / 24, (1 - torch.cos(th)) / th ** 2)
    E = torch.eye(3, dtype=torch.float64) + A * K + B * (K @ K)
    Rn = E @ P[:, :, :3]
    on = P[:, :, 3] + tau
    img_t = torch.as_tensor(np.asarray(img, np.int64))
    d = (Rn[img_t] @ t64(dirs)[:, :, None])[:, :, 0]
    o = on[img_t]
    ra = np.asarray(rays_a)
    rows, owner = [], []
    for r, s, c in ra:
        rows.extend(range(s, s + c))
        owner.extend([r] * c)
    rows, owner = torch.as_tensor(rows, dtype=torch.int64), torch.as_tensor(owner, dtype=torch.int64)
    x = o[owner] + t64(ts)[rows][:, None] * d[owner]
    L = (t64(dx)[rows] * x).sum()
    L.backward()
    return np.concatenate([w.grad.numpy(), tau.grad.numpy()], 1)
