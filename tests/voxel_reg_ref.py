"""fp64 restatement of the voxel-grid regularisers (DESIGN.md §6d, ngp_voxel_reg in include/ngp_b200.h), the per-element
bound the kernel's fp32 result is judged by, and a numpy fp32 copy of the kernel (with optional planted mistakes) that
lets the CPU suite show the bound rejects wrong kernels.

Everything here works on the node block B cut out of the fields: V[lo_x:hi_x, lo_y:hi_y, lo_z:hi_z, C].  Inside that
block a forward difference whose neighbour lies outside B is 0, so the block alone defines the losses."""
import math

import numpy as np
import torch

EPS_TV = 1e-8
U = 2.0 ** -24           # unit round-off of fp32


def block_of(t, block):
    """The block B of a field [G, G, G, C] (torch or numpy)."""
    lx, ly, lz, hx, hy, hz = block
    return t[lx:hx, ly:hy, lz:hz]


def _diffs(V):
    """Forward differences along x, y, z of a block [nx, ny, nz, C]; 0 on the last slice of each axis."""
    dx, dy, dz = torch.zeros_like(V), torch.zeros_like(V), torch.zeros_like(V)
    dx[:-1] = V[1:] - V[:-1]
    dy[:, :-1] = V[:, 1:] - V[:, :-1]
    dz[:, :, :-1] = V[:, :, 1:] - V[:, :, :-1]
    return dx, dy, dz


def reference(sh_b, den_b, weights, n_nodes=None):
    """fp64 autograd of L = w_tv_sigma L_tv_sigma + w_tv_sh L_tv_sh + w_sparsity L_sparsity over the block.  Returns
    (L, dL/dsh_b, dL/dden_b, A_sh, A_den): A is the per-element magnitude the bound scales with (see bound()).
    n_nodes = |B| when the arguments are only a slab of B (default: the block given is B)."""
    w_sig, w_sh, w_sp = (float(w) for w in weights)
    S = sh_b.double().clone().requires_grad_(True)
    P = den_b.double().clone().requires_grad_(True)
    N = P[..., 0].numel() if n_nodes is None else n_nodes

    def tv(V):
        dx, dy, dz = _diffs(V)
        return torch.sqrt(dx * dx + dy * dy + dz * dz + EPS_TV)

    r = torch.relu(P)
    L = (w_sig * tv(P).sum() / N + w_sh * tv(S).sum() / (N * S.shape[-1])
         + w_sp * torch.log1p(2 * r * r).sum() / N)
    gS, gP = torch.autograd.grad(L, (S, P))
    with torch.no_grad():
        A_sh = w_sh / (N * S.shape[-1]) * tv_magnitude(S.detach())
        A_den = w_sig / N * tv_magnitude(P.detach()) + w_sp / N * (4 * r / (1 + 2 * r * r)).detach()
    return float(L.detach()), gS, gP, A_sh, A_den


def tv_magnitude(V):
    """T(v) = (|Dx| + |Dy| + |Dz|)(v) / s(v) + sum_a |D_a(v - e_a)| / s(v - e_a): the sum of the absolute values of
    the terms the kernel adds up for the TV gradient of v (its own and its three backward neighbours')."""
    dx, dy, dz = _diffs(V)
    s = torch.sqrt(dx * dx + dy * dy + dz * dz + EPS_TV)
    T = (dx.abs() + dy.abs() + dz.abs()) / s
    T[1:] += (dx.abs() / s)[:-1]
    T[:, 1:] += (dy.abs() / s)[:, :-1]
    T[:, :, 1:] += (dz.abs() / s)[:, :, :-1]
    return T


def bound(pre, g, A, scale):
    """Per-element bound on |out - (pre + scale * g)|, g the fp64 gradient, A its magnitude from reference().
    The kernel's fp32 TV term: each difference of two fp32 values rounds once (u); a square adds 2u + u, the sum of
    three squares and eps (rounded to fp32) 3 more: s^2 within 6u, s within 4u after the sqrt.  Own term: the sum of
    three differences 3u, the division u: 8u of |term|; a neighbour term 6u; adding up to four terms 3u of their
    absolute sum.  So the TV sum is within 11u T.  The sparsity derivative 4r / (1 + 2r^2) costs 4u of itself.  The
    weight / |B| is rounded to fp32 (u), then one multiply each by the weight and the scale and one add of the two
    parts (3u); the accumulation into pre rounds once more: u |pre + scale g|.  16u covers 11u + 4u plus higher
    orders; the whole gets a factor 1.5 of head-room."""
    return 1.5 * (U * (pre + scale * g).abs() + 16 * U * scale * A)


def loss_bound(terms_sum, n_blocks, w_sp):
    """Bound on |loss_kernel - L|: every term c s carries 6u of itself (c 2u, s 4u), the fp32 sum adds at most
    (2 + 5 + 8 + n_blocks) roundings of the total (per thread, warp tree, block sum, one atomic per block); a sparsity
    term log(fl(1 + 2r^2)) is off by up to u + one ulp absolutely (q rounds by u relative), i.e. 3u w_sp / |B| per
    node, 3u w_sp in all.  terms_sum = the fp64 L (every term is >= 0).  Factor 2 of head-room."""
    return 2.0 * (U * (6 + 15 + n_blocks) * terms_sum + 3 * U * w_sp)


def check(out_sh, out_den, pre_sh, pre_den, sh_b, den_b, weights, scale, what="", n_nodes=None, first_x=0):
    """Compare the kernel's block results with pre + scale * the fp64 gradient; raises AssertionError naming the worst
    element.  Returns (L_fp64, worst error / bound).  For a slab of B (n_nodes = |B|) whose first x-slice is not B's,
    first_x = 1 leaves out that slice, whose gradient needs the slice before it."""
    L, gS, gP, A_sh, A_den = reference(sh_b, den_b, weights, n_nodes)
    worst = 0.0
    for name, out, pre, g, A in (("sh", out_sh, pre_sh, gS, A_sh), ("density", out_den, pre_den, gP, A_den)):
        out, pre, g, A = out[first_x:], pre[first_x:], g[first_x:], A[first_x:]
        pre64 = pre.double()
        want = pre64 + scale * g
        err = (out.double() - want).abs()
        b = bound(pre64, g, A, scale)
        ratio = torch.where(b > 0, err / b, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
        r = float(ratio.max())
        if r > 1:
            idx = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
            bad = int((ratio > 1).sum())
            raise AssertionError(f"{what}: {name} gradient of {bad} elements off the fp64 bound; worst at {idx}: got "
                                 f"{float(out[idx]):.9e} want {float(want[idx]):.9e} err {float(err[idx]):.3e} "
                                 f"bound {float(b[idx]):.3e}")
        worst = max(worst, r)
    return L, worst


# ---- numpy fp32 copy of the kernel ----------------------------------------------------------------------------------
FAULTS = ("drop_neighbour", "eps_outside_sqrt", "block_off_by_one", "relu_on_tv")


def kernel_np(sh, den, block, weights, scale, dsh, dden, fault=None):
    """The kernel's arithmetic in numpy fp32 on full fields sh [G,G,G,3D], den [G,G,G,1], accumulating into dsh / dden
    in place.  fault plants one mistake: drop_neighbour (the z backward neighbour's term is lost), eps_outside_sqrt
    (s = sqrt(D^2) + eps), block_off_by_one (the x forward difference of B's last slice reads the node after B),
    relu_on_tv (the density TV is taken of ReLU(density))."""
    f32 = np.float32
    G = sh.shape[0]
    lo, hi = np.array(block[:3]), np.array(block[3:])
    if fault == "block_off_by_one":
        hi_x = min(hi[0] + 1, G)
    else:
        hi_x = hi[0]
    N = float(np.prod(hi - lo))
    w_sig, w_sh, w_sp = (float(w) for w in weights)
    eps = f32(EPS_TV)

    def norm(a, b, c):
        q = (a * a + b * b) + c * c
        if fault == "eps_outside_sqrt":
            return np.sqrt(q) + eps
        return np.sqrt(q + eps)

    def tv_grad(F):
        """F: full field [G,G,G,C] fp32 -> TV gradient term t on B (fp32), the kernel's order of operations."""
        nx, ny, nz = hi - lo
        gi = np.arange(lo[0], hi[0])[:, None, None, None]
        gj = np.arange(lo[1], hi[1])[None, :, None, None]
        gk = np.arange(lo[2], hi[2])[None, None, :, None]
        z = f32(0)

        def shifted(di, dj, dk):
            """V(v + (di, dj, dk)) on B; entries whose node lies outside the grid are 0 (never used)."""
            out = np.zeros((nx, ny, nz, F.shape[-1]), np.float32)
            i0, j0, k0 = lo + np.array([di, dj, dk])
            si = slice(max(i0, 0), min(i0 + nx, G))
            sj = slice(max(j0, 0), min(j0 + ny, G))
            sk = slice(max(k0, 0), min(k0 + nz, G))
            src = F[si, sj, sk]
            out[si.start - i0:si.start - i0 + src.shape[0], sj.start - j0:sj.start - j0 + src.shape[1],
                sk.start - k0:sk.start - k0 + src.shape[2]] = src
            return out

        v0 = shifted(0, 0, 0)
        px, py, pz = gi + 1 < hi_x, gj + 1 < hi[1], gk + 1 < hi[2]
        mx, my, mz = gi > lo[0], gj > lo[1], gk > lo[2]
        dx = np.where(px, shifted(1, 0, 0) - v0, z)
        dy = np.where(py, shifted(0, 1, 0) - v0, z)
        dz = np.where(pz, shifted(0, 0, 1) - v0, z)
        s = norm(dx, dy, dz)
        t = -((dx + dy) + dz) / s
        b = shifted(-1, 0, 0)
        ex, ey, ez = v0 - b, np.where(py, shifted(-1, 1, 0) - b, z), np.where(pz, shifted(-1, 0, 1) - b, z)
        t = np.where(mx, t + ex / norm(ex, ey, ez), t)
        b = shifted(0, -1, 0)
        ex, ey, ez = np.where(px, shifted(1, -1, 0) - b, z), v0 - b, np.where(pz, shifted(0, -1, 1) - b, z)
        t = np.where(my, t + ey / norm(ex, ey, ez), t)
        if fault != "drop_neighbour":
            b = shifted(0, 0, -1)
            ex, ey, ez = np.where(px, shifted(1, 0, -1) - b, z), np.where(py, shifted(0, 1, -1) - b, z), v0 - b
            t = np.where(mz, t + ez / norm(ex, ey, ez), t)
        return t.astype(np.float32)

    sl = tuple(slice(a, b) for a, b in zip(lo, hi))
    if w_sh != 0:
        c = f32(w_sh / (N * sh.shape[-1]))
        dsh[sl] = dsh[sl] + f32(scale) * (c * tv_grad(sh))
    if w_sig != 0 or w_sp != 0:
        g = np.zeros(tuple(hi - lo) + (1,), np.float32)
        if w_sig != 0:
            F = np.maximum(den, f32(0)) if fault == "relu_on_tv" else den
            g = f32(w_sig / N) * tv_grad(F)
        if w_sp != 0:
            r = np.maximum(den[sl], f32(0))
            q = f32(1) + f32(2) * (r * r)
            g = g + f32(w_sp / N) * ((f32(4) * r) / q)
        dden[sl] = dden[sl] + f32(scale) * g
