"""The voxel-grid kernels (csrc/voxel.cu) against fp64 on inputs they have to round: the shipped lattice (G = 256,
radius 0.0125, so neither the spacing nor c_min is a power of two), G = 97, 2 and 1 at non-dyadic spacings, positions
from a real march, uniform over the lattice and a few ulp either side of node planes; a field past 2^31 floats;
non-finite, far and edge positions with the fields and gradients passed as views between guard bands; degenerate
directions; device row counts in both forward modes.  tests/test_gpu_voxel_grid.py keeps the exact-arithmetic inputs on which sigma must be bit-exact.

Per-element bound of the forward (fwd_ref), term by term.  With u = (x - c_min) / radius in fp64 (x, c_min and radius
the fp32 values the kernel takes), the kernel's u_hat = fl(fl(x - c_min) / radius) has |u_hat - u| <= 2 eps (1 + eps)
|u| per axis, plus eps where u < 0 (the fraction u_hat + 1 of a cell in (-1, 0) rounds).  The masked trilinear field
is continuous and piecewise trilinear, so moving from u to u_hat changes every channel by at most
sum_axis du_axis * L_axis, L_axis the largest |difference of adjacent nodes| along that axis over the cells the box
[u - du, u + du] touches (outside nodes count as 0).  This holds whether or not floor(u_hat) = floor(u), so no sample
is excluded.  On top, the fp32 arithmetic at u_hat: each corner weight carries <= 5 roundings (1 - fraction and two
products), the product w f one more and the 8-term sum 7, so the interpolated channel is off by <= 14 eps A,
A = sum_q w_q |f_q|.  sigma = ReLU is 1-Lipschitz.  rgb: z = sum_k Y_k v_k with Y_k carrying <= 16 roundings of 1.1
(the fp32 normalisation of d and the products) and the k-sum D+1 roundings of |Y_k v_k|; sigmoid is 1/4-Lipschitz and
adds <= 4 roundings.  A factor 2 covers second-order terms (A and |v| taken at u, not u_hat).

Backward (bwd_ref): the ReLU mask is the fp64 one except where |density_fp64| is within the sigma bound; there the
kernel's own mask (sigma_kernel > 0, which is what its backward reads) is the reference's (voxel_ref.grads
relu_mask).  The kernel scatters fl(w(u_hat) g_kernel) onto the corners of u_hat's cell, the reference w(u) g onto
u's.  A node's trilinear weight is a tent function, 1-Lipschitz per axis, so |w_n(u_hat) - w_n(u)| <= dU = sum du,
and any node the kernel may touch lies in the cells of [u - du, u + du] (the extended touched set; nothing outside it
may be written).  g_kernel is off by dg (the rgb bound through s(1 - s) plus the products, as in
test_gpu_voxel_grid); the weight and the product add 6 eps; the atomic sum (cnt - 1) eps of the sum of |terms|.

The CPU tests at the end run the comparator on a numpy fp32 restatement of the kernels with one planted mistake each
(fractions quantised to 1/16 or rounded to fp16, c_min shifted by radius/2, radius at fp16 precision, an out-of-grid
corner clamped to the edge node, a corner's weight given to its x-neighbour): each is rejected, in the forward and in
the backward, while fp64 rounded to fp32 and the fault-free restatement pass.  test_dyadic_inputs_hide_quantised_
fractions shows why the exact-arithmetic suite cannot see the first mistake."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

import voxel_ref as R
from composite_ref import U, np_composite_f64, termination_window
from taichi_nerfs_b200.layout import make_voxel_layout

DEV = "cuda"
EPS = 2.0 ** -24          # unit round-off of fp32
CHUNK = 8192
CONFIGS = [(256, 0.0125, 2), (97, 0.03, 1), (2, 0.3, 0), (1, 0.0125, 2)]
_OFFS = torch.tensor([(a, b, c) for a in range(3) for b in range(3) for c in range(3)])     # [27, 3]


def _report(what, d):
    print("voxel-fp64", what, json.dumps(d))


# ---- fp64 reference and bounds ---------------------------------------------------------------------------------------
def _u(xyz, lay):
    return (xyz.double() - lay.c_min) / lay.radius


def _du(u):
    """Per axis: |u_hat - u| for the kernel's fp32 u_hat (module doc)."""
    return 2 * EPS * (1 + EPS) * u.abs() + EPS * (u < 0).double()


def _box_nodes(u, du, G):
    """The nodes of every cell [u - du, u + du] touches: base = floor(u - du) per axis, offsets 0..span+1 (span 0 or
    1) -> node [n, 27] (-1 outside the grid), in-box [n, 27] (offset <= span + 1 on every axis), span [n, 3]."""
    base = torch.floor(u - du)
    span = torch.floor(u + du) - base
    assert bool((span <= 1).all()), "a position error wider than a cell"
    base = base.clamp(-4, G + 4).long()
    idx = base[:, None, :] + _OFFS[None]
    inside = ((idx >= 0) & (idx < G)).all(-1)
    node = torch.where(inside, (idx[..., 0] * G + idx[..., 1]) * G + idx[..., 2], torch.full_like(idx[..., 0], -1))
    inbox = (_OFFS[None] <= span.long()[:, None, :] + 1).all(-1)
    return node, inbox, span.long(), idx


def _position_term(field, u, du):
    """[n, C]: sum_axis du_axis * L_axis over the cells [u - du, u + du] touches (module doc)."""
    G, Cn = field.shape[0], field.shape[-1]
    node, _, span, _ = _box_nodes(u, du, G)
    V = R.gather(field, node).reshape(-1, 3, 3, 3, Cn)
    out = torch.zeros(u.shape[0], Cn, dtype=torch.float64)
    for ax in range(3):
        diff = (V.narrow(1 + ax, 1, 2) - V.narrow(1 + ax, 0, 2)).abs()
        valid = []
        for k in range(3):
            ar = torch.arange(2 if k == ax else 3)
            valid.append(ar[None, :] <= span[:, k:k + 1] + (0 if k == ax else 1))
        m = valid[0][:, :, None, None] & valid[1][:, None, :, None] & valid[2][:, None, None, :]
        L = torch.where(m[..., None], diff, torch.zeros_like(diff)).amax(dim=(1, 2, 3))
        out += du[:, ax:ax + 1] * L
    return out


def fwd_ref(xyz, dirs, sh, den, lay):
    """fp64 sigma, rgb, the pre-ReLU density and the per-element bounds b_sigma [N], b_rgb [N, 3] (module doc).  xyz,
    dirs: fp32 CPU tensors; the fields anywhere (only the corners of the samples are gathered)."""
    deg = lay.sh_degree
    D = (deg + 1) ** 2
    parts = []
    for s in range(0, xyz.shape[0], CHUNK):
        x, d = xyz[s:s + CHUNK], dirs[s:s + CHUNK]
        u = _u(x, lay)
        du = _du(u)
        node, w = R.corners(x, lay.grid, lay.radius, lay.c_min)
        vals = torch.cat([R.gather(sh, node), R.gather(den, node)], -1)
        sigma, rgb = R._model(w, vals, d, deg)
        v = (w[..., None] * vals).sum(1)
        A = (w[..., None] * vals.abs()).sum(1)
        pos = torch.cat([_position_term(sh, u, du), _position_term(den, u, du)], -1)
        dv = pos + 14 * EPS * A
        dd = d.double() / torch.norm(d.double(), dim=1, keepdim=True)
        Y = R.sh_basis(deg, dd).abs()[:, None, :]
        dvs = dv[:, :3 * D].reshape(-1, 3, D)
        vs = v[:, :3 * D].reshape(-1, 3, D).abs() + dvs
        dz = (Y * dvs).sum(-1) + EPS * (16 * 1.1 * vs.sum(-1) + (D + 1) * (Y * vs).sum(-1))
        parts.append(dict(sigma=sigma, rgb=rgb, pre=v[:, -1], b_sigma=2 * dv[:, -1], b_rgb=2 * (0.25 * dz + 4 * EPS)))
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}


def check_fwd(sigma, rgb, ref, what):
    """-> the largest error / bound of sigma and rgb.  NaN fails."""
    out = {}
    for name, got, want, b in (("sigma", sigma, ref["sigma"], ref["b_sigma"]), ("rgb", rgb, ref["rgb"], ref["b_rgb"])):
        err = (got.double().cpu() - want).abs()
        bad = ~(err <= b)
        if bool(bad.any()):
            i = int(bad.flatten().nonzero()[0])
            raise AssertionError(f"{what}: {name} of {int(bad.sum())} elements off, first flat {i}: err "
                                 f"{float(err.flatten()[i]):.3e} bound {float(b.flatten()[i]):.3e}")
        out[name] = float((err / b.clamp(min=1e-300)).max()) if err.numel() else 0.0
    return out


def bwd_ref(xyz, dirs, sh, den, lay, dsig, drgb, ref, sigma_kernel):
    """The fp64 gradient and its per-element bound on the extended touched set (module doc): -> (nodes [U] sorted,
    want [U, 3D + 1], tol [U, 3D + 1]); channels are the sh channels then the density."""
    deg, G = lay.sh_degree, lay.grid
    D = (deg + 1) ** 2
    amb = ref["pre"].abs() <= ref["b_sigma"]
    mask = torch.where(amb, sigma_kernel.double().cpu() > 0, ref["pre"] > 0)
    nodes, gsh, gden = R.grads(xyz, dirs, sh, den, lay.radius, deg, dsig, drgb, lay.c_min, relu_mask=mask)
    n = xyz.shape[0]
    d = dirs.double() / torch.norm(dirs.double(), dim=1, keepdim=True)
    Y = R.sh_basis(deg, d)[:, None, :]
    s = ref["rgb"][:, :, None]
    dr = drgb.double()[:, :, None]
    g_sh = (dr * (s * (1 - s)) * Y).reshape(n, 3 * D)
    dg_sh = (dr.abs() * (Y.abs() * (ref["b_rgb"][:, :, None] + 3 * EPS) + 0.25 * 16 * 1.1 * EPS)).reshape(n, 3 * D)
    dg_sh = dg_sh + 3 * EPS * g_sh.abs()
    g = torch.cat([g_sh, (dsig.double() * mask)[:, None]], 1).abs()
    dg = torch.cat([dg_sh, torch.zeros(n, 1, dtype=torch.float64)], 1)
    rows_n, rows_t1, rows_t2 = [], [], []
    for c0 in range(0, n, CHUNK):
        sl = slice(c0, c0 + CHUNK)
        u = _u(xyz[sl], lay)
        du = _du(u)
        node, inbox, _, idx = _box_nodes(u, du, G)
        w = (1 - (u[:, None, :] - idx.double()).abs()).clamp(min=0).prod(-1)       # exact tent weight at u
        dU = du.sum(1)[:, None, None]
        Wb = (w[..., None] + dU)
        gg, dgg = g[sl][:, None, :], dg[sl][:, None, :]
        t1 = Wb * (dgg + 6 * EPS * gg) + dU * (gg + dgg)
        t2 = Wb * gg
        ok = inbox & (node >= 0)
        rows_n.append(node[ok])
        rows_t1.append(t1.expand(-1, 27, -1)[ok])
        rows_t2.append(t2.expand(-1, 27, -1)[ok])
    rn = torch.cat(rows_n)
    ext, inv = torch.unique(rn, return_inverse=True)
    Cn = 3 * D + 1
    t1 = torch.zeros(len(ext), Cn, dtype=torch.float64).index_add_(0, inv, torch.cat(rows_t1))
    t2 = torch.zeros(len(ext), Cn, dtype=torch.float64).index_add_(0, inv, torch.cat(rows_t2))
    cnt = torch.zeros(len(ext), 1, dtype=torch.float64).index_add_(0, inv, torch.ones(len(rn), 1, dtype=torch.float64))
    want = torch.zeros(len(ext), Cn, dtype=torch.float64)
    pos = torch.searchsorted(ext, nodes)
    assert bool((ext[pos] == nodes).all())
    want[pos] = torch.cat([gsh, gden], 1)
    return ext, want, t1 + cnt * EPS * t2


def check_bwd(got, want, tol, what):
    """got [U, 3D + 1] (the kernel's gradient at the extended touched set) -> the largest error / bound."""
    err = (got.double().cpu() - want).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i, j = [int(v) for v in bad.nonzero()[0]]
        raise AssertionError(f"{what}: gradient of {int(bad.sum())} floats off, first node row {i} channel {j}: got "
                             f"{float(got[i, j]):.6e} want {float(want[i, j]):.6e} tol {float(tol[i, j]):.3e}")
    assert float(want.abs().max()) > 0
    return float((err / tol.clamp(min=1e-300)).max())


def _kernel_grad_rows(dsh, dden, nodes):
    D3 = dsh.shape[-1]
    it = nodes.to(dsh.device)
    return torch.cat([dsh.reshape(-1, D3)[it], dden.reshape(-1, 1)[it]], 1).cpu()


def _written_outside(dsh, dden, nodes):
    """Nodes outside `nodes` with a non-zero gradient (the buffers start at zero)."""
    D3 = dsh.shape[-1]
    nz = (dsh.reshape(-1, D3) != 0).any(1) | (dden.reshape(-1) != 0)
    nz[nodes.to(nz.device)] = False
    return int(nz.sum())


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _march_points(O, n_rays, seed):
    """Samples of a training march (random noise) of Lego-shaped rays through the scene box at scale 0.5, every
    occupancy bit set."""
    from oracle.train_step import make_rays
    o, d = make_rays(n_rays, seed=seed)
    hits = O.ray_aabb_intersect(o, d, 0.5)
    noise = np.random.default_rng(seed).random(n_rays, dtype=np.float32)
    bits = np.full(128 ** 3 // 8, 255, np.uint8)
    return O.raymarching_train(o, d, hits, bits, noise, 1, 0.5, 0.0, 128, 1024)[1]


def _uniform_points(rng, n, lay):
    """Uniform fp32 points over the lattice span widened by two cells on every side."""
    lo, hi = lay.c_min - 2 * lay.radius, lay.c_min + (lay.grid + 1) * lay.radius
    return rng.uniform(lo, hi, (n, 3)).astype(np.float32)


def _plane_points(rng, n, lay):
    """Every coordinate within 4 fp32 ulp of a node plane (nodes -1..G), on either side."""
    i = rng.integers(-1, lay.grid + 1, (n, 3))
    p = (lay.c_min + i * float(lay.radius)).astype(np.float32)
    k = rng.integers(-4, 5, (n, 3)).astype(np.float32)
    return (p + k * np.spacing(np.abs(p))).astype(np.float32)


def _directions(rng, n):
    """Arbitrary fp32 vectors: normal components scaled by 10^[-3, 3]."""
    return (rng.standard_normal((n, 3)) * 10.0 ** rng.uniform(-3, 3, (n, 1))).astype(np.float32)


def _device_fields(seed, G, deg, lo=-1.0, hi=1.0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    sh = torch.empty(G, G, G, 3 * (deg + 1) ** 2, device=DEV).uniform_(-1, 1, generator=gen)
    den = torch.empty(G, G, G, 1, device=DEV).uniform_(lo, hi, generator=gen)
    return sh, den


def _grads_in(rng, n):
    dsig = rng.standard_normal(n).astype(np.float32)
    drgb = rng.standard_normal((n, 3)).astype(np.float32)
    dsig[::7] = 0
    drgb[3::11] = 0
    return torch.from_numpy(dsig), torch.from_numpy(drgb)


# ---- 1. arbitrary fp32 inputs at non-dyadic lattices ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("G,radius,deg", CONFIGS)
def test_arbitrary_inputs_vs_fp64(oracle, G, radius, deg):
    """Forward and both backward mappings against fp64 within the per-element bound of the module doc, on march,
    uniform and near-plane positions, arbitrary directions and signed fields; nothing outside the extended touched set
    is written."""
    from taichi_nerfs_b200 import ops
    lay = make_voxel_layout(G, radius, deg)
    cl = lay.as_ctypes()
    rng = np.random.default_rng(G * 10 + deg)
    x = np.concatenate([_march_points(oracle, 24, G + deg), _uniform_points(rng, 20000, lay),
                        _plane_points(rng, 8000, lay)])
    xyz = torch.from_numpy(x)
    dirs = torch.from_numpy(_directions(rng, x.shape[0]))
    S, P = _device_fields(G * 10 + deg, G, deg)
    X, Dd = xyz.to(DEV), dirs.to(DEV)
    sigma, rgb = ops.voxel_fwd(X, Dd, S, P, cl)
    ref = fwd_ref(xyz, dirs, S, P, lay)
    rf = check_fwd(sigma, rgb, ref, f"G={G} deg={deg}")
    assert G == 1 or (bool((ref["pre"] > 0).any()) and bool((ref["pre"] < 0).any()))   # G = 1: one node
    # the fp32 cell differs from the fp64 one for some near-plane samples
    u = _u(xyz, lay)
    uh = torch.from_numpy(((x - np.float32(lay.c_min)) / np.float32(lay.radius)).astype(np.float64))
    moved = int((torch.floor(uh) != torch.floor(u)).any(1).sum())
    assert moved > 0 or G <= 2
    dsig, drgb = _grads_in(rng, x.shape[0])
    nodes, want, tol = bwd_ref(xyz, dirs, S, P, lay, dsig, drgb, ref, sigma)
    rb = {}
    for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
        dsh, dden = torch.zeros_like(S), torch.zeros_like(P)
        ops.voxel_bwd(X, Dd, sigma, rgb, dsig.to(DEV), drgb.to(DEV), cl, dsh, dden, mapping=mapping)
        rb[mapping] = check_bwd(_kernel_grad_rows(dsh, dden, nodes), want, tol, f"G={G} deg={deg} mapping={mapping}")
        assert _written_outside(dsh, dden, nodes) == 0, "a node outside the extended touched set was written"
    _report(f"G={G} r={radius} deg={deg}", dict(samples=x.shape[0], cell_moved=moved, fwd=rf, bwd_warp=rb[0],
                                                 bwd_thread=rb[1], nodes=int(len(nodes))))


# ---- 2. a field past 2^31 floats ------------------------------------------------------------------------------------
def _count_not(t, value, chunk=1 << 28):
    return sum(int((t[s:s + chunk] != value).sum()) for s in range(0, t.numel(), chunk))


@pytest.mark.gpu
def test_field_past_2_pow_31_floats():
    """G = 432, degree 2: the sh field holds 432^3 * 27 = 2,176,782,336 floats.  Samples in cells whose nodes have
    node * 27 >= 2^31 (x-index >= 427), near node 0, and in cells straddling 2^31 (x-index 426, y about 80).  One
    buffer holds [guard, dsh, sh]: 2^31 sentinel floats in front of dsh and dsh in front of sh, so every address an
    int32 wrap of node * 27 would reach lies in this buffer; the guard must stay bit-unchanged.  Forward and both
    backward mappings against fp64 at the touched nodes; every other gradient float stays zero."""
    from taichi_nerfs_b200 import ops
    G, deg = 432, 2
    lay = make_voxel_layout(G, 0.0125, deg)
    cl = lay.as_ctypes()
    Cn = 27
    n_sh = G ** 3 * Cn
    assert n_sh > 2 ** 31
    guard = 2 ** 31
    need = (guard + 2 * n_sh + 2 * G ** 3) * 4 + (4 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    rng = np.random.default_rng(432)
    n = 6000
    u_hi = np.stack([rng.uniform(427, 432, n), rng.uniform(-1, G, n), rng.uniform(-1, G, n)], 1)
    u_lo = rng.uniform(-1, 2, (n, 3))
    u_st = np.stack([rng.uniform(426, 427, n), rng.uniform(79, 81, n), rng.uniform(0, G, n)], 1)
    x = (lay.c_min + np.concatenate([u_hi, u_lo, u_st]) * lay.radius).astype(np.float32)
    xyz = torch.from_numpy(x)
    dirs = torch.from_numpy(_directions(rng, x.shape[0]))
    node, _ = R.corners(xyz, G, lay.radius, lay.c_min)
    high = (node * Cn >= 2 ** 31)
    assert bool(high.any()) and bool((node == 0).any())
    assert bool((high.any(1) & ((node >= 0) & ~high).any(1)).any()), "no cell straddles 2^31"
    torch.cuda.reset_peak_memory_stats()
    buf = P = dden = None
    try:
        buf = torch.empty(guard + 2 * n_sh, device=DEV)
        front = buf[:guard]
        front.fill_(7.0)
        dsh = buf[guard:guard + n_sh].view(G, G, G, Cn)
        dsh.zero_()
        S = buf[guard + n_sh:].view(G, G, G, Cn)
        gen = torch.Generator(device=DEV).manual_seed(432)
        S.uniform_(-1, 1, generator=gen)
        P = torch.empty(G, G, G, 1, device=DEV).uniform_(-1, 1, generator=gen)
        dden = torch.zeros_like(P)
        X, Dd = xyz.to(DEV), dirs.to(DEV)
        sigma, rgb = ops.voxel_fwd(X, Dd, S, P, cl)
        ref = fwd_ref(xyz, dirs, S, P, lay)
        rf = check_fwd(sigma, rgb, ref, "G=432")
        dsig, drgb = _grads_in(rng, x.shape[0])
        nodes, want, tol = bwd_ref(xyz, dirs, S, P, lay, dsig, drgb, ref, sigma)
        assert int((nodes * Cn >= 2 ** 31).sum()) > 0
        rb = {}
        for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
            ops.voxel_bwd(X, Dd, sigma, rgb, dsig.to(DEV), drgb.to(DEV), cl, dsh, dden, mapping=mapping)
            rb[mapping] = check_bwd(_kernel_grad_rows(dsh, dden, nodes), want, tol, f"G=432 mapping={mapping}")
            it = nodes.to(DEV)
            dsh.view(-1, Cn)[it] = 0
            dden.view(-1)[it] = 0
            assert _count_not(dsh.view(-1), 0.0) == 0 and _count_not(dden.view(-1), 0.0) == 0, \
                "a gradient float no sample reaches was written"
            assert _count_not(front, 7.0) == 0, "the floats an int32 wrap of node * 27 would reach were written"
        peak = torch.cuda.max_memory_allocated()
        _report("G=432 deg=2", dict(fwd=rf, bwd_warp=rb[0], bwd_thread=rb[1], nodes=int(len(nodes)),
                                    nodes_above_2_31=int((nodes * Cn >= 2 ** 31).sum()),
                                    peak_gib=round(peak / 2 ** 30, 2)))
    finally:
        del buf, P, dden
        torch.cuda.empty_cache()


# ---- 3. non-finite, far and degenerate inputs -----------------------------------------------------------------------
PAD = 4099
SENT = -12345.0


def _guarded(shape, fill):
    n = math.prod(shape)
    buf = torch.full((n + 2 * PAD,), fill, device=DEV)
    return buf, buf[PAD:PAD + n].view(*shape)


def _guards_intact(buf, fill):
    g = torch.cat([buf[:PAD], buf[-PAD:]])
    if math.isnan(fill):
        return bool(torch.isnan(g).all())
    return bool((g.view(torch.int32) == torch.tensor([fill], device=DEV).view(torch.int32)).all())


def _x_at(lay, u):
    """The fp32 x nearest c_min + u * radius whose kernel u_hat = fl(fl(x - c_min) / radius) is exactly u (searched
    within 4096 ulp; the lattice of the edge test is chosen so that one exists for every u asked for)."""
    f32 = np.float32
    x0 = f32(lay.c_min + u * float(lay.radius))
    k = np.arange(-4096, 4097)
    xs = (x0 + k * np.spacing(x0)).astype(f32)
    hit = np.flatnonzero(((xs - f32(lay.c_min)) / f32(lay.radius)).astype(np.float64) == u)
    assert hit.size, f"no fp32 x gives u_hat = {u} exactly"
    return xs[hit[np.argmin(np.abs(k[hit]))]]


def _edge_positions(lay, rng):
    """Interior base points with one axis or all three set to: u = -1, in (-1, 0), G-1, in (G-1, G), G; the float
    below c_min and the float above c_min + (G-1) radius.  And points with NaN, +-inf, +-1e30 on one axis or all."""
    G = lay.grid
    f32 = np.float32
    top = float(lay.c_min) + (G - 1) * float(lay.radius)
    above = f32(top) if float(f32(top)) > top else np.nextafter(f32(top), f32(np.inf))
    coords = [_x_at(lay, -1.0), _x_at(lay, -0.5), f32(lay.c_min + (-1 + 1e-4) * lay.radius),
              f32(lay.c_min + -1e-3 * lay.radius), _x_at(lay, G - 1.0), _x_at(lay, G - 0.5),
              f32(lay.c_min + (G - 1e-4) * lay.radius), _x_at(lay, float(G)),
              np.nextafter(f32(lay.c_min), f32(-np.inf)), above]
    special = [np.nan, np.inf, -np.inf, 1e30, -1e30]

    def spread(vals):
        pts = []
        for v in vals:
            for axes in ([0], [1], [2], [0, 1, 2]):
                p = (lay.c_min + (rng.uniform(0, G - 1, 3)) * lay.radius).astype(np.float32)
                p[axes] = v
                pts.append(p)
        return np.array(pts, np.float32)
    return spread(coords), spread(special)


def _call_bwd(X, Dd, sigma, rgb, dsig, drgb, cl, dsh, dden, mapping, found=None):
    from taichi_nerfs_b200 import _lib, ops
    p = ops._ptr
    _lib.check(_lib.load().ngp_voxel_bwd(p(X), p(Dd), p(sigma), p(rgb), p(dsig), p(drgb), C.byref(cl), p(dsh),
                                         p(dden), X.shape[0], p(found), int(mapping), ops._stream()))


@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2])
def test_nonfinite_far_and_edge_positions_with_guard_bands(deg):
    """Fields between NaN guard bands, gradients between sentinel bands.  Fully masked samples (NaN, +-inf, +-1e30 on
    any axis) give sigma = 0 and rgb = 0.5 bit for bit and scatter nothing; edge positions (u = -1, G-1, G, the
    floats just outside the lattice) match fp64; no guard is read (outputs finite) or written (bit-unchanged)."""
    from taichi_nerfs_b200 import ops
    G = 7
    lay = make_voxel_layout(G, 0.037, deg)   # u = -1, -0.5, G-1, G-0.5, G are exact kernel u_hat
    cl = lay.as_ctypes()
    D3 = 3 * (deg + 1) ** 2
    rng = np.random.default_rng(70 + deg)
    edge, special = _edge_positions(lay, rng)
    gen = torch.Generator(device=DEV).manual_seed(deg)
    sh_buf, S = _guarded((G, G, G, D3), math.nan)
    den_buf, P = _guarded((G, G, G, 1), math.nan)
    S.uniform_(-1, 1, generator=gen)
    P.uniform_(-1, 1, generator=gen)
    for pts, masked in ((special, True), (np.concatenate([edge, special]), False)):
        xyz = torch.from_numpy(pts)
        dirs = torch.from_numpy(rng.standard_normal(pts.shape).astype(np.float32))
        X, Dd = xyz.to(DEV), dirs.to(DEV)
        sigma, rgb = ops.voxel_fwd(X, Dd, S, P, cl)
        assert bool(torch.isfinite(sigma).all()) and bool(torch.isfinite(rgb).all()), "a guard band was read"
        if masked:
            assert bool((sigma == 0).all()) and bool((rgb == 0.5).all()), "a fully masked sample is not sigma 0, rgb 0.5"
        else:
            fin = np.flatnonzero(np.isfinite(pts).all(1) & (np.abs(pts) < 1e29).all(1))
            assert fin.size == edge.shape[0]
            it = torch.from_numpy(fin)
            ref = fwd_ref(xyz[it], dirs[it], S, P, lay)
            check_fwd(sigma[it.to(DEV)], rgb[it.to(DEV)], ref, f"edge positions deg={deg}")
            assert bool((ref["sigma"] != 0).any())
            dsig, drgb = _grads_in(rng, len(fin))
            nodes, want, tol = bwd_ref(xyz[it], dirs[it], S, P, lay, dsig, drgb, ref, sigma[it.to(DEV)])
        gs = torch.from_numpy(rng.standard_normal(pts.shape[0]).astype(np.float32)) + 2
        gr = torch.from_numpy(rng.standard_normal((pts.shape[0], 3)).astype(np.float32)) + 2
        if not masked:   # the edge rows get the gradients of the reference; the masked rows keep theirs
            gs[it], gr[it] = dsig, drgb
        for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
            dsh_buf, dsh = _guarded((G, G, G, D3), SENT)
            dden_buf, dden = _guarded((G, G, G, 1), SENT)
            dsh.zero_()
            dden.zero_()
            found = torch.zeros(1, device=DEV, dtype=torch.int32)
            _call_bwd(X, Dd, sigma, rgb, gs.to(DEV), gr.to(DEV), cl, dsh, dden, mapping, found)
            assert _guards_intact(dsh_buf, SENT) and _guards_intact(dden_buf, SENT), "a gradient guard was written"
            assert int(found) == 0
            if masked:
                assert not bool(dsh.any()) and not bool(dden.any()), "a fully masked sample scattered"
            else:
                check_bwd(_kernel_grad_rows(dsh, dden, nodes), want, tol, f"edge positions deg={deg} map={mapping}")
                assert _written_outside(dsh, dden, nodes) == 0
    assert _guards_intact(sh_buf, math.nan) and _guards_intact(den_buf, math.nan)


def _degenerate_dirs():
    """(kind, direction) rows: zero, subnormal, components whose squares overflow fp32."""
    rows = [("zero", (0.0, 0.0, 0.0)), ("zero", (-0.0, 0.0, -0.0)),
            ("subnormal", (1e-40, -3e-41, 2e-39)), ("subnormal", (1e-45, 0.0, 0.0)),
            ("subnormal", (-1e-45, 1e-45, 0.0)), ("subnormal", (3e-39, 2e-39, -1e-39)),
            ("huge", (1e30, -2e30, 5e29)), ("huge", (3e38, 3e38, -3e38)), ("huge", (0.0, -1e30, 0.0)),
            ("huge", (1e30, 1e-30, 0.0)), ("tiny", (1e-20, 3e-20, -2e-20))]
    return [k for k, _ in rows], np.array([d for _, d in rows], np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2])
def test_degenerate_directions(deg):
    """Subnormal and ~1e30 directions match fp64 (the kernel scales them by a power of two before squaring).  A zero
    direction: at degree 0 rgb is finite and matches fp64; at degree >= 1 rgb is NaN, as voxel_ref's 0/0 gives, and
    the backward writes NaN into the sh gradient exactly where voxel_ref's is NaN and raises found_inf."""
    from taichi_nerfs_b200 import ops
    G = 9
    lay = make_voxel_layout(G, 0.03, deg)
    cl = lay.as_ctypes()
    rng = np.random.default_rng(deg)
    kinds, dd = _degenerate_dirs()
    reps = 16
    kinds = kinds * reps
    dirs = torch.from_numpy(np.tile(dd, (reps, 1)))
    n = dirs.shape[0]
    xyz = torch.from_numpy((lay.c_min + rng.uniform(0.2, G - 1.2, (n, 3)) * lay.radius).astype(np.float32))
    S, P = _device_fields(90 + deg, G, deg, lo=0.1, hi=1.0)
    X, Dd = xyz.to(DEV), dirs.to(DEV)
    sigma, rgb = ops.voxel_fwd(X, Dd, S, P, cl)
    zero = torch.tensor([k == "zero" for k in kinds])
    ref = fwd_ref(xyz, dirs, S, P, lay)
    check_fwd(sigma, sigma, dict(sigma=ref["sigma"], rgb=ref["sigma"], b_sigma=ref["b_sigma"],
                                 b_rgb=ref["b_sigma"]), "sigma")
    if deg == 0:
        check_fwd(sigma, rgb, ref, "deg 0")
    else:
        assert bool(torch.isnan(rgb.cpu()[zero]).all()) and bool(torch.isnan(ref["rgb"][zero]).all())
        fin = torch.from_numpy(np.flatnonzero(~zero.numpy()))
        sub = {k: v[fin] for k, v in ref.items()}
        check_fwd(sigma[fin.to(DEV)], rgb[fin.to(DEV)], sub, f"deg {deg} non-zero directions")
    dsig = torch.ones(n)
    drgb = torch.from_numpy(rng.standard_normal((n, 3)).astype(np.float32)) + 3
    for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
        dsh, dden = torch.zeros_like(S), torch.zeros_like(P)
        found = torch.zeros(1, device=DEV, dtype=torch.int32)
        ops.voxel_bwd(X, Dd, sigma, rgb, dsig.to(DEV), drgb.to(DEV), cl, dsh, dden, found, mapping)
        nodes, gsh, gden = R.grads(xyz, dirs, S, P, lay.radius, deg, dsig, drgb, lay.c_min)
        got = dsh.reshape(-1, dsh.shape[-1])[nodes.to(DEV)].cpu()
        assert torch.equal(torch.isnan(got), torch.isnan(gsh)), "NaN gradient pattern differs from voxel_ref"
        assert int(found) == (1 if deg >= 1 else 0)
        assert bool(torch.isfinite(dden).all())
    if deg >= 1:   # without the zero directions, the full comparison
        keep = torch.from_numpy(np.flatnonzero(~zero.numpy()))
        x2, d2 = xyz[keep], dirs[keep]
        X2, D2 = x2.to(DEV), d2.to(DEV)
        s2, c2 = ops.voxel_fwd(X2, D2, S, P, cl)
        ref2 = fwd_ref(x2, d2, S, P, lay)
        nodes, want, tol = bwd_ref(x2, d2, S, P, lay, dsig[keep], drgb[keep], ref2, s2)
        for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
            dsh, dden = torch.zeros_like(S), torch.zeros_like(P)
            found = torch.zeros(1, device=DEV, dtype=torch.int32)
            ops.voxel_bwd(X2, D2, s2, c2, dsig[keep].to(DEV), drgb[keep].to(DEV), cl, dsh, dden, found, mapping)
            assert int(found) == 0
            check_bwd(_kernel_grad_rows(dsh, dden, nodes), want, tol, f"degenerate dirs deg={deg} map={mapping}")


# ---- 4. device row counts -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2])
def test_device_row_count_both_modes(deg):
    """ngp_voxel_fwd_dyn, full and density-only, with *n_dev in {0, 1, 31, 32, 33, n_max-1, n_max, n_max+5, -3} and
    n_max = 1001 (not a multiple of any block's sample count): rows below min(n_max, max(n_dev, 0)) equal the static
    call bit for bit (density-only: its sigma), every row from there on keeps its sentinel."""
    from taichi_nerfs_b200 import _lib, ops
    G = 13
    lay = make_voxel_layout(G, 0.03, deg)
    cl = lay.as_ctypes()
    rng = np.random.default_rng(13 + deg)
    n_max, pad = 1001, 37
    X = torch.from_numpy(_uniform_points(rng, n_max + pad, lay)).to(DEV)
    Dd = torch.from_numpy(_directions(rng, n_max + pad)).to(DEV)
    S, P = _device_fields(130 + deg, G, deg)
    s_all, c_all = ops.voxel_fwd(X[:n_max].contiguous(), Dd[:n_max].contiguous(), S, P, cl)
    assert bool((s_all > 0).any())
    bits = lambda t: t.view(torch.int32)   # noqa: E731
    p = ops._ptr
    lib = _lib.load()
    for nd in (0, 1, 31, 32, 33, n_max - 1, n_max, n_max + 5, -3):
        m = min(max(nd, 0), n_max)
        n_dev = torch.tensor([nd], device=DEV, dtype=torch.int32)
        sig = torch.full((n_max + pad,), -7.0, device=DEV)
        rgb = torch.full((n_max + pad, 3), -7.0, device=DEV)
        _lib.check(lib.ngp_voxel_fwd_dyn(p(X), p(Dd), p(S), p(P), C.byref(cl), p(sig), p(rgb), n_max, p(n_dev),
                                         ops._stream()))
        assert torch.equal(bits(sig[:m]), bits(s_all[:m])) and torch.equal(bits(rgb[:m]), bits(c_all[:m])), nd
        assert bool((sig[m:] == -7).all()) and bool((rgb[m:] == -7).all()), f"n_dev={nd}: a row past the count"
        sig1 = torch.full((n_max + pad,), -7.0, device=DEV)
        _lib.check(lib.ngp_voxel_fwd_dyn(p(X), None, None, p(P), C.byref(cl), p(sig1), None, n_max, p(n_dev),
                                         ops._stream()))
        assert torch.equal(bits(sig1[:m]), bits(s_all[:m])), f"n_dev={nd}: density-only sigma differs"
        assert bool((sig1[m:] == -7).all()), f"n_dev={nd}: density-only wrote a row past the count"


# ---- 5. an svox frame against an fp64 frame -------------------------------------------------------------------------
FRAME_RAYS = 6000
THR = 1e-4


def _frame_ref(sig, rgb, b_sig, b_rgb, deltas, ts, rays_a, n_active):
    """fp64 opacity, depth and rgb (white background) of every ray compositing its first n_active samples, and the
    per-pixel bound: 2 x (the first-order effect of the per-sample bounds: sum_s mag_s b_sigma_s with mag the
    compositing's sum of |terms| of d(output)/d(sigma_s), plus sum_s w_s b_rgb_s) + the compositing's own fp32 error,
    8 u (N + 4) of (|output| + 1) (each transmittance factor and weight carries a few u of T_s absolutely)."""
    n, S = rays_a.shape[0], sig.size
    z, zs, z3 = np.zeros(n), np.zeros(S), np.zeros((n, 3))
    one = np.ones(n)
    base = np_composite_f64(sig, rgb, deltas, ts, rays_a, THR, one, z, z3, zs, n_active=n_active)
    act = base["active"]
    ray_of = np.empty(S, np.int64)
    for r, s0, cnt in rays_a:
        ray_of[s0:s0 + cnt] = r

    def per_ray(v):
        return np.bincount(ray_of, weights=np.where(act, v, 0.0), minlength=n)
    cnt = rays_a[:, 2].astype(np.float64)
    comp = 8 * U * (cnt + 4)
    op, dep, out = base["op"], base["dep"], base["rgb"] + (1 - base["op"])[:, None]
    b_op = 2 * per_ray(base["mag"] * b_sig) + comp * (op + 1)
    tmax = np.zeros(n)
    np.maximum.at(tmax, ray_of, ts.astype(np.float64))
    mag_d = np_composite_f64(sig, rgb, deltas, ts, rays_a, THR, z, one, z3, zs, n_active=n_active)["mag"]
    b_dep = 2 * per_ray(mag_d * b_sig) + comp * (dep + tmax)
    b_out = np.zeros((n, 3))
    for c in range(3):
        gr = np.zeros((n, 3))
        gr[:, c] = 1
        mag_c = np_composite_f64(sig, rgb, deltas, ts, rays_a, THR, -one, z, gr, zs, n_active=n_active)["mag"]
        b_out[:, c] = 2 * (per_ray(mag_c * b_sig) + per_ray(base["w"] * b_rgb[:, c])) + comp * (np.abs(out[:, c]) + 2)
    return dict(op=op, dep=dep, rgb=out, b_op=b_op, b_dep=b_dep, b_rgb=b_out)


def _frame_model():
    """VoxelGrid(G = 40, radius 0.027, degree 2) with random fields (signed densities) and occupancy."""
    from modules.voxel_grid import VoxelGrid
    m = VoxelGrid(grid_size=40, grid_radius=0.027, sh_degree=2).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(40)
    with torch.no_grad():
        m.sh_fields.uniform_(-1, 1, generator=gen)
        m.density_fields.uniform_(-10, 30, generator=gen)
        bits = (torch.rand(m.density_bitfield.shape[0], 8, device=DEV, generator=gen) < 0.85).to(torch.uint8)
        m.density_bitfield.copy_((bits << torch.arange(8, device=DEV, dtype=torch.uint8)).sum(1).to(torch.uint8))
    return m.eval()


@pytest.mark.gpu
def test_svox_frame_vs_fp64_frame(oracle):
    """render(test_time=True) of a VoxelGrid (G = 40, radius 0.027, degree 2, random fields and occupancy) against a
    frame built outside the library: the oracle's zero-noise march, voxel_ref.forward in fp64, the compositing in fp64
    with T_threshold 1e-4 and 1024 samples per ray.  A ray whose termination index is ambiguous (its fp64
    transmittance is within the fp32 error of the threshold, widened by the sigma bound: composite_ref.
    termination_window at sigma +- b_sigma) passes if it matches the fp64 frame at any admissible index; every other
    ray at the fp64 index.  More than 2^21 samples, so the module forward runs in several chunks."""
    from modules.rendering import render
    from oracle.train_step import make_rays
    m = _frame_model()
    o, d = make_rays(FRAME_RAYS, seed=40)
    with torch.no_grad(), torch.autocast('cuda', dtype=torch.float16):
        out = render(m, torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), test_time=True)
    got_op, got_dep, got_rgb = [out[k].float().cpu().numpy().astype(np.float64) for k in ("opacity", "depth", "rgb")]
    hits = oracle.ray_aabb_intersect(o, d, m.scale)
    rays_a, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, m.density_bitfield.cpu().numpy(),
                                                                 np.zeros(FRAME_RAYS, np.float32), m.cascades,
                                                                 m.scale, 0.0, m.grid_size, 1024)
    assert int(out["total_samples"]) == S and S > 2 ** 21, S
    ref = fwd_ref(torch.from_numpy(xyzs), torch.from_numpy(dirs), m.sh_fields.detach(), m.density_fields.detach(),
                  m._layout)
    sig, rgb = ref["sigma"].numpy(), ref["rgb"].numpy()
    b_sig, b_rgb = ref["b_sigma"].numpy(), ref["b_rgb"].numpy()
    n_lo = termination_window(sig + b_sig, deltas, rays_a, THR)[0]
    n_hi = termination_window(np.maximum(sig - b_sig, 0), deltas, rays_a, THR)[1]
    n_lo, n_hi = np.minimum(n_lo, n_hi), np.maximum(n_lo, n_hi)
    ambiguous = n_lo < n_hi
    ok = np.zeros(FRAME_RAYS, bool)
    ratio = 0.0
    for j in range(int((n_hi - n_lo).max()) + 1):
        with np.errstate(divide="ignore"):   # np_composite_f64's conditioning factor of rays with sigma = 0 (unused)
            f = _frame_ref(sig, rgb, b_sig, b_rgb, deltas, ts, rays_a, np.minimum(n_lo + j, n_hi))
        err = np.stack([np.abs(got_op - f["op"]), np.abs(got_dep - f["dep"])] + [np.abs(got_rgb[:, c] - f["rgb"][:, c])
                                                                                for c in range(3)], 1)
        b = np.stack([f["b_op"], f["b_dep"]] + [f["b_rgb"][:, c] for c in range(3)], 1)
        # a ray without samples has opacity and depth 0 exactly and a zero depth bound: 0 / 0 counts as 0
        r = np.where(err == 0, 0.0, err / np.where(b > 0, b, 1e-300)).max(1)
        if j == 0:
            ratio = float(r[~ambiguous].max())
        ok |= r <= 1
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, f"{bad.size} pixels off the fp64 frame, first ray {bad[0]} (ambiguous: {ambiguous[bad[0]]})"
    terminated = int((n_hi < rays_a[:, 2]).sum())
    assert 0 < terminated < FRAME_RAYS and bool((rays_a[:, 2] == 0).any())
    _report("frame", dict(rays=FRAME_RAYS, samples=S, ambiguous=int(ambiguous.sum()), terminated=terminated,
                          empty_rays=int((rays_a[:, 2] == 0).sum()),
                          max_err_over_bound=ratio))


# ---- CPU: the comparator accepts fp64 rounded to fp32 and rejects the planted mistakes ------------------------------
FAULTS = ["fraction_1_16", "fraction_fp16", "c_min_half_cell", "radius_fp16", "edge_clamped", "weight_to_x_neighbour"]
_Y = [0.28209479177387814, 0.4886025119029199, 1.0925484305920792, 0.31539156525252005, 0.5462742152960396]


def _np_cells(x, lay, fault=None):
    """The kernel's cell arithmetic in fp32 numpy -> node [N, 8] (-1 masked), weight [N, 8] fp32."""
    f32 = np.float32
    G = lay.grid
    c_min, r = f32(lay.c_min), f32(lay.radius)
    if fault == "c_min_half_cell":
        c_min = f32(c_min + r / f32(2))
    if fault == "radius_fp16":
        r = f32(np.float16(r))
    u = (x - c_min) / r
    fl = np.floor(u)
    fr = (u - fl).astype(f32)
    if fault == "fraction_1_16":
        fr = (np.floor(fr * f32(16)) / f32(16)).astype(f32)
    if fault == "fraction_fp16":
        fr = fr.astype(np.float16).astype(f32)
    ok = (fl >= -1) & (fl < G)
    lo = np.where(ok, fl, -2).astype(np.int64)
    nodes, ws = [], []
    for q in range(8):
        bits = np.array([(q >> 2) & 1, (q >> 1) & 1, q & 1])
        idx = lo + bits
        w3 = [fr[:, k] if bits[k] else (f32(1) - fr[:, k]).astype(f32) for k in range(3)]
        ws.append(((w3[0] * w3[1]).astype(f32) * w3[2]).astype(f32))
        inside = ((idx >= 0) & (idx < G)).all(1)
        if fault == "edge_clamped":
            inside = (lo > -2).all(1)
            idx = np.clip(idx, 0, G - 1)
        nodes.append(np.where(inside, (idx[:, 0] * G + idx[:, 1]) * G + idx[:, 2], -1))
    node, w = np.stack(nodes, 1), np.stack(ws, 1)
    if fault == "weight_to_x_neighbour":
        w[:, 4] = (w[:, 4] + w[:, 0]).astype(f32)
        w[:, 0] = 0
    return node, w


def _np_basis(d, deg):
    f32 = np.float32
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    Y0, Y1, Ya, Yb, Yc = [f32(c) for c in _Y]
    cols = [np.full_like(x, Y0)]
    if deg >= 1:
        cols += [-Y1 * y, Y1 * z, -Y1 * x]
    if deg >= 2:
        cols += [Ya * (x * y), -Ya * (y * z), Yb * (f32(2) * (z * z) - x * x - y * y), -Ya * (x * z),
                 Yc * (x * x - y * y)]
    return np.stack(cols, 1).astype(f32)


def _np_dir(d):
    norm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return (d / norm[:, None]).astype(np.float32)


def np_fwd(x, dirs, sh, den, lay, fault=None):
    """The forward in fp32 numpy, in the kernel's operation order, with one planted mistake."""
    f32 = np.float32
    deg, D = lay.sh_degree, lay.sh_dim
    node, w = _np_cells(x, lay, fault)
    F = np.concatenate([sh.reshape(-1, 3 * D), den.reshape(-1, 1)], 1)
    v = np.zeros((x.shape[0], 3 * D + 1), f32)
    for q in range(8):
        ok = node[:, q] >= 0
        v[ok] = (v[ok] + (w[ok, q, None] * F[node[ok, q]]).astype(f32)).astype(f32)
    Y = _np_basis(_np_dir(dirs), deg)
    part = (v[:, :3 * D].reshape(-1, 3, D) * Y[:, None, :]).astype(f32)
    z = np.zeros((x.shape[0], 3), f32)
    for k in range(D):
        z = (z + part[:, :, k]).astype(f32)
    rgb = (f32(1) / (f32(1) + np.exp(-z))).astype(f32)
    return np.maximum(v[:, -1], f32(0)), rgb


def np_bwd(x, dirs, sigma, rgb, dsig, drgb, lay, fault=None):
    """The backward in fp32 numpy (np.add.at: sequential atomics) -> dsh [G^3, 3D], dden [G^3, 1]."""
    f32 = np.float32
    deg, D, G = lay.sh_degree, lay.sh_dim, lay.grid
    node, w = _np_cells(x, lay, fault)
    Y = _np_basis(_np_dir(dirs), deg)
    gcol = (drgb * (rgb * (f32(1) - rgb)).astype(f32)).astype(f32)
    g = np.concatenate([(gcol[:, :, None] * Y[:, None, :]).reshape(-1, 3 * D),
                        np.where(sigma > 0, dsig, f32(0))[:, None]], 1).astype(f32)
    out = np.zeros((G ** 3, 3 * D + 1), f32)
    for q in range(8):
        ok = node[:, q] >= 0
        np.add.at(out, node[ok, q], (w[ok, q, None] * g[ok]).astype(f32))
    return out[:, :-1], out[:, -1:]


@pytest.fixture(scope="module", params=[(97, 0.03, 1), (24, 0.0125, 2)], ids=["G97deg1", "G24deg2"])
def cpu_case(request):
    G, radius, deg = request.param
    lay = make_voxel_layout(G, radius, deg)
    rng = np.random.default_rng(G + deg)
    x = np.concatenate([_uniform_points(rng, 5000, lay), _plane_points(rng, 2000, lay)])
    dirs = _directions(rng, x.shape[0])
    sh = rng.uniform(-1, 1, (G, G, G, 3 * lay.sh_dim)).astype(np.float32)
    den = rng.uniform(-1, 1, (G, G, G, 1)).astype(np.float32)
    dsig, drgb = _grads_in(rng, x.shape[0])
    xt, dt, St, Pt = (torch.from_numpy(a) for a in (x, dirs, sh, den))
    ref = fwd_ref(xt, dt, St, Pt, lay)
    sigma, rgb = np_fwd(x, dirs, sh, den, lay)
    nodes, want, tol = bwd_ref(xt, dt, St, Pt, lay, dsig, drgb, ref, torch.from_numpy(sigma))
    return dict(lay=lay, x=x, dirs=dirs, sh=sh, den=den, dsig=dsig.numpy(), drgb=drgb.numpy(), ref=ref,
                sigma=sigma, rgb=rgb, nodes=nodes, want=want, tol=tol)


def _np_check_bwd(case, dsh, dden, what):
    rows = torch.from_numpy(np.concatenate([dsh, dden], 1))
    nz = (rows != 0).any(1)
    nz[case["nodes"]] = False
    assert not bool(nz.any()), f"{what}: a node outside the extended touched set was written"
    return check_bwd(rows[case["nodes"]], case["want"], case["tol"], what)


def test_comparator_accepts_fp64_rounded_and_numpy_fp32(cpu_case):
    c = cpu_case
    ref = c["ref"]
    assert bool((ref["pre"] > 0).any()) and bool((ref["pre"] < 0).any())
    check_fwd(ref["sigma"].float(), ref["rgb"].float(), ref, "fp64 rounded to fp32")
    check_fwd(torch.from_numpy(c["sigma"]), torch.from_numpy(c["rgb"]), ref, "numpy fp32")
    want32 = c["want"].float()
    check_bwd(want32, c["want"], c["tol"], "fp64 gradient rounded to fp32")
    dsh, dden = np_bwd(c["x"], c["dirs"], c["sigma"], c["rgb"], c["dsig"], c["drgb"], c["lay"])
    _np_check_bwd(c, dsh, dden, "numpy fp32")


@pytest.mark.parametrize("fault", FAULTS)
def test_comparator_rejects_forward(cpu_case, fault):
    c = cpu_case
    sigma, rgb = np_fwd(c["x"], c["dirs"], c["sh"], c["den"], c["lay"], fault)
    with pytest.raises(AssertionError):
        check_fwd(torch.from_numpy(sigma), torch.from_numpy(rgb), c["ref"], fault)


@pytest.mark.parametrize("fault", FAULTS)
def test_comparator_rejects_backward(cpu_case, fault):
    c = cpu_case
    dsh, dden = np_bwd(c["x"], c["dirs"], c["sigma"], c["rgb"], c["dsig"], c["drgb"], c["lay"], fault)
    with pytest.raises(AssertionError):
        _np_check_bwd(c, dsh, dden, fault)


def test_dyadic_inputs_hide_quantised_fractions():
    """On the exact-arithmetic inputs of test_gpu_voxel_grid (power-of-two spacing, u on a 1/16 grid) a kernel that
    quantises its fractions to 1/16 computes what the correct kernel computes, bit for bit, so that suite cannot see
    it; on the inputs here it is rejected (test_comparator_rejects_*[fraction_1_16])."""
    from test_gpu_voxel_grid import _positions, _radius
    for G, deg in ((97, 1), (2, 0)):
        lay = make_voxel_layout(G, _radius(G), deg)
        rng = np.random.default_rng(G)
        x = _positions(rng, 3000, G, lay).numpy()
        dirs = rng.standard_normal(x.shape).astype(np.float32)
        sh = rng.uniform(-1, 1, (G, G, G, 3 * lay.sh_dim)).astype(np.float32)
        den = (rng.integers(-8, 9, (G, G, G, 1)) / 8).astype(np.float32)
        a, b = np_fwd(x, dirs, sh, den, lay), np_fwd(x, dirs, sh, den, lay, "fraction_1_16")
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        g = np_bwd(x, dirs, a[0], a[1], np.ones(x.shape[0], np.float32), np.ones((x.shape[0], 3), np.float32), lay)
        h = np_bwd(x, dirs, a[0], a[1], np.ones(x.shape[0], np.float32), np.ones((x.shape[0], 3), np.float32), lay,
                   "fraction_1_16")
        assert np.array_equal(g[0], h[0]) and np.array_equal(g[1], h[1])
