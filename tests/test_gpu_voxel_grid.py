"""The voxel-grid model (`--model_name svox`) on the GPU: forward and field backward against the fp64 restatement
(tests/voxel_ref.py) for degrees 0-2 and G = 256, 97, 2 with both backward mappings, the density-only mode, the inf
flag, one NGPTrainer step against torch's Adam, train.main end to end and test-time rendering.

Inputs are chosen so that the lattice mapping is exact in fp32: the node spacing is a power of two and every position
is c_min + u * radius with u on a 1/16 grid, so u, the fraction in the cell and every corner weight (three factors of
5 significant bits) are exact.  Densities are multiples of 1/8 in [-1, 1]: w * density then has at most 19 significant
bits and the 8-term sum stays exact, so sigma (and with it the ReLU mask) must equal fp64 bit for bit.  The sh
coefficients are arbitrary fp32; their error bounds are written out where they are used."""
import math

import numpy as np
import pytest
import torch

import voxel_ref as R
from taichi_nerfs_b200.layout import make_voxel_layout

pytestmark = pytest.mark.gpu

DEV = "cuda"
EPS = 2.0 ** -24          # unit round-off of fp32


def _radius(G):
    return {256: 2.0 ** -6, 97: 2.0 ** -5, 2: 0.25}[G]


def _positions(rng, n, G, lay, same_cell=False):
    """World points c_min + u * radius, u on a 1/16 grid: random over [-3, G+2) (inside and outside the field, inside
    and outside the scene box [-0.5, 0.5]^3), lattice nodes, and points on the faces of the last cell (u = G-1)."""
    if same_cell:
        u = 10 % G + rng.integers(0, 16, (n, 3)) / 16.0
    else:
        u = rng.integers(-3 * 16, (G + 2) * 16, (n, 3)) / 16.0
        nodes = rng.integers(0, G, (256, 3)).astype(np.float64)
        face = rng.integers(0, (G - 1) * 16, (256, 3)) / 16.0
        face[np.arange(256), rng.integers(0, 3, 256)] = G - 1
        u = np.concatenate([u, nodes, face, [[G - 1] * 3, [0, 0, 0], [G, G, G], [-1, -1, -1]]])
    x = lay.c_min + u * lay.radius
    assert np.array_equal(x.astype(np.float32).astype(np.float64), x)
    return torch.from_numpy(x.astype(np.float32))


def _fields(seed, G, deg):
    """sh uniform in [-1, 1), densities multiples of 1/8 in [-1, 1]; on the GPU (1.8 GB at G = 256, degree 2)."""
    D = (deg + 1) ** 2
    gen = torch.Generator(device=DEV).manual_seed(seed)
    sh = torch.rand(G, G, G, 3 * D, device=DEV, generator=gen) * 2 - 1
    den = torch.randint(-8, 9, (G, G, G, 1), device=DEV, generator=gen).float() / 8
    return sh, den


def _rgb_bound(xyz, dirs, sh, radius, c_min, deg):
    """Per-element bound on |rgb - rgb_fp64|.  z = sum_k Y_k v_k with v_k = sum_q w_q sh_q (w exact): each v_k carries
    <= 9 roundings of the terms w|sh| (A_k = interpolation of |sh|), each Y_k <= 16 roundings of its size (the fp32
    normalisation of d and the products, |Y_k| <= 1.1), the k-sum <= D+1 roundings of |Y_k v_k|.  sigmoid is
    1/4-Lipschitz and costs <= 4 roundings of itself (expf, add, div).  Factor 2 of head-room on the whole."""
    D = (deg + 1) ** 2
    node, w = R.corners(xyz, sh.shape[0], radius, c_min)
    vals = R.gather(sh, node)
    d = dirs.double() / torch.norm(dirs.double(), dim=1, keepdim=True)
    Y = R.sh_basis(deg, d).abs()[:, None, :]
    A = (w[..., None] * vals.abs()).sum(1).reshape(-1, 3, D)
    v = (w[..., None] * vals).sum(1).reshape(-1, 3, D).abs()
    dz = EPS * (9 * (Y * A).sum(-1) + 16 * 1.1 * v.sum(-1) + (D + 1) * (Y * v).sum(-1))
    return 2 * (0.25 * dz + 4 * EPS)


def _check_fwd_bwd(G, deg, xyz, dirs, S, P, mapping):
    """xyz, dirs on the CPU; the fields S, P on the GPU."""
    from taichi_nerfs_b200 import ops
    lay = make_voxel_layout(G, _radius(G), deg)
    cl = lay.as_ctypes()
    n = xyz.shape[0]
    X, Dd = xyz.to(DEV), dirs.to(DEV)
    sigma, rgb = ops.voxel_fwd(X, Dd, S, P, cl)
    s_ref, c_ref = R.forward(xyz, dirs, S, P, lay.radius, deg, lay.c_min)
    assert torch.equal(sigma.cpu().double(), s_ref)                          # exact by construction (module doc)
    assert bool((s_ref > 0).any()) and bool((R.interpolate(xyz, P, lay.radius, lay.c_min) < 0).any())
    bound = _rgb_bound(xyz, dirs, S, lay.radius, lay.c_min, deg)
    err = (rgb.cpu().double() - c_ref).abs()
    assert bool((err <= bound).all()), float((err - bound).max())
    # density-only mode: the forward's sigma bit for bit
    assert torch.equal(ops.voxel_fwd(X, None, None, P, cl), sigma)

    rng = np.random.default_rng(n + G)
    dsig = torch.from_numpy(rng.standard_normal(n).astype(np.float32))
    drgb = torch.from_numpy(rng.standard_normal((n, 3)).astype(np.float32))
    dsig[::7] = 0           # rows with zero gradient issue nothing
    dsh = torch.zeros_like(S)
    dden = torch.zeros_like(P)
    ops.voxel_bwd(X, Dd, sigma, rgb, dsig.to(DEV), drgb.to(DEV), cl, dsh, dden, mapping=mapping)
    nodes, gsh, gden = R.grads(xyz, dirs, S, P, lay.radius, deg, dsig, drgb, lay.c_min)
    D = (deg + 1) ** 2
    k_sh = dsh.reshape(-1, 3 * D)
    k_den = dden.reshape(-1, 1)
    # nothing is written outside the nodes the batch touches
    written = (k_sh != 0).any(1) | (k_den != 0).any(1)
    assert bool(torch.isin(written.nonzero().squeeze(1).cpu(), nodes).all())
    k_sh, k_den = k_sh[nodes.to(DEV)].cpu().double(), k_den[nodes.to(DEV)].cpu().double()
    node, w = R.corners(xyz, G, lay.radius, lay.c_min)
    idx = R.touched_nodes(node)

    def scatter(per_sample):       # sum over samples of w_q * per_sample at the touched nodes
        return R.scatter(node, w[..., None] * per_sample[:, None, :], idx)

    cnt = R.scatter(node, torch.ones(n, 8, 1, dtype=torch.float64), idx)   # contributions per node
    # density: g = dsigma * (sigma > 0) exactly (the mask is exact); only the atomic sum rounds: (n-1) eps sum|terms|
    g_den = torch.where(s_ref > 0, dsig.double(), torch.zeros_like(s_ref))[:, None]
    tol_den = cnt * EPS * scatter(g_den.abs())
    assert bool(((k_den - gden).abs() <= tol_den).all())
    # sh: g = drgb_c * s(1-s) * Y_k from the kernel's fp32 rgb.  |d s(1-s)/ds| <= 1, so the fp32 rgb error (bound
    # above) plus 3 roundings moves s(1-s) by <= bound + 3 eps; Y_k carries <= 16 roundings of 1.1; the two products
    # 3 more of |g|.  Then the atomic sum: (n-1) eps sum |w g|.
    d = dirs.double() / torch.norm(dirs.double(), dim=1, keepdim=True)
    Y = R.sh_basis(deg, d)[:, None, :]
    s = c_ref[:, :, None]
    dr = drgb.double().abs()[:, :, None]
    g = (dr * (s * (1 - s)) * Y.abs()).reshape(n, 3 * D)
    dg = (dr * (Y.abs() * (bound[:, :, None] + 3 * EPS) + 0.25 * 16 * 1.1 * EPS)).reshape(n, 3 * D) + 3 * EPS * g
    tol_sh = scatter(dg) + cnt * EPS * scatter(g)
    err = (k_sh - gsh).abs()
    assert bool((err <= tol_sh).all()), float((err - tol_sh).max())
    assert float(gsh.abs().max()) > 0


@pytest.mark.parametrize("deg", [0, 1, 2])
@pytest.mark.parametrize("G", [256, 97, 2])
def test_forward_backward_vs_fp64(G, deg):
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(G * 10 + deg)
    lay = make_voxel_layout(G, _radius(G), deg)
    xyz = _positions(rng, 20001, G, lay)           # not a multiple of any block's sample count
    dirs = torch.from_numpy(rng.standard_normal((xyz.shape[0], 3)).astype(np.float32))
    sh, den = _fields(G * 10 + deg, G, deg)
    for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
        _check_fwd_bwd(G, deg, xyz, dirs, sh, den, mapping)


@pytest.mark.parametrize("deg", [0, 2])
def test_backward_colliding_atomics(deg):
    """8000 samples in one cell: every reduction of the batch lands on the same 8 nodes."""
    from taichi_nerfs_b200 import ops
    G = 97
    rng = np.random.default_rng(deg)
    lay = make_voxel_layout(G, _radius(G), deg)
    xyz = _positions(rng, 8000, G, lay, same_cell=True)
    dirs = torch.from_numpy(rng.standard_normal((8000, 3)).astype(np.float32))
    sh, den = _fields(deg, G, deg)
    for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
        _check_fwd_bwd(G, deg, xyz, dirs, sh, den, mapping)


def test_empty_batch_and_device_count():
    from taichi_nerfs_b200 import _lib, ops
    import ctypes as C
    lay = make_voxel_layout(16, 0.125, 1)
    cl = lay.as_ctypes()
    sh = torch.rand(16, 16, 16, 12, device=DEV)
    den = torch.rand(16, 16, 16, 1, device=DEV)
    e = torch.zeros(0, 3, device=DEV)
    s, c = ops.voxel_fwd(e, e, sh, den, cl)
    assert s.shape == (0,) and c.shape == (0, 3)
    dsh, dden = torch.zeros_like(sh), torch.zeros_like(den)
    ops.voxel_bwd(e, e, s, c, s, c, cl, dsh, dden)
    assert not dsh.any() and not dden.any()
    # _dyn: rows >= *n_dev untouched
    x = (torch.rand(1000, 3, device=DEV) - 0.5)
    d = torch.randn(1000, 3, device=DEV)
    sig = torch.full((1000,), -7.0, device=DEV)
    rgb = torch.full((1000, 3), -7.0, device=DEV)
    n_dev = torch.tensor([617], device=DEV, dtype=torch.int32)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(_lib.load().ngp_voxel_fwd_dyn(p(x), p(d), p(sh), p(den), C.byref(cl), p(sig), p(rgb), 1000, p(n_dev),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    s_all, c_all = ops.voxel_fwd(x, d, sh, den, cl)
    assert torch.equal(sig[:617], s_all[:617]) and torch.equal(rgb[:617], c_all[:617])
    assert bool((sig[617:] == -7).all()) and bool((rgb[617:] == -7).all())


def test_found_inf_flag():
    from taichi_nerfs_b200 import ops
    lay = make_voxel_layout(16, 0.125, 2)
    cl = lay.as_ctypes()
    sh = torch.rand(16, 16, 16, 27, device=DEV)
    den = torch.rand(16, 16, 16, 1, device=DEV)
    x = (torch.rand(500, 3, device=DEV) - 0.5)
    d = torch.randn(500, 3, device=DEV)
    s, c = ops.voxel_fwd(x, d, sh, den, cl)
    for mapping in (ops.VOXEL_BWD_WARP, ops.VOXEL_BWD_THREAD):
        found = torch.zeros(1, device=DEV, dtype=torch.int32)
        ds, dc = torch.ones_like(s), torch.ones_like(c)
        ops.voxel_bwd(x, d, s, c, ds, dc, cl, torch.zeros_like(sh), torch.zeros_like(den), found, mapping)
        assert int(found) == 0
        dc[123, 1] = math.inf
        ops.voxel_bwd(x, d, s, c, ds, dc, cl, torch.zeros_like(sh), torch.zeros_like(den), found, mapping)
        assert int(found) == 1


def test_module_autograd_and_refusals():
    """VoxelGrid.forward returns fp32 under fp16 autocast; its backward equals the kernel's; positions that require
    grad are refused; an unsupported degree raises."""
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200 import ops
    m = VoxelGrid(grid_size=32, grid_radius=0.05, origin_sh=0.0).to(DEV)
    with torch.no_grad():
        m.sh_fields.uniform_(-1, 1)
        m.density_fields.uniform_(-1, 1)
    x = (torch.rand(3000, 3, device=DEV) - 0.5) * 1.2
    d = torch.randn(3000, 3, device=DEV)
    with torch.autocast('cuda', dtype=torch.float16):
        sigma, rgb = m(x.half(), d.half())
    assert sigma.dtype == torch.float32 and rgb.dtype == torch.float32
    (sigma.sum() + rgb.sum()).backward()
    s2, c2 = ops.voxel_fwd(x.half().float(), d.half().float(), m.sh_fields.detach(), m.density_fields.detach(),
                           m._clayout)
    dsh, dden = torch.zeros_like(m.sh_fields), torch.zeros_like(m.density_fields)
    ops.voxel_bwd(x.half().float(), d.half().float(), s2, c2, torch.ones_like(s2), torch.ones_like(c2), m._clayout,
                  dsh, dden)
    assert torch.equal(sigma, s2) and torch.equal(rgb, c2)
    torch.testing.assert_close(m.sh_fields.grad, dsh, rtol=0, atol=1e-4)     # atomic order only
    torch.testing.assert_close(m.density_fields.grad, dden, rtol=0, atol=1e-4)
    assert torch.equal(m.density(x), ops.voxel_fwd(x, None, None, m.density_fields.detach(), m._clayout))
    with pytest.raises(NotImplementedError):
        m(x.requires_grad_(True), d)
    with pytest.raises(ValueError):
        VoxelGrid(sh_degree=3, grid_size=4)


def test_trainer_step_equals_torch_adam():
    """NGPTrainer over a VoxelGrid: the backward scatters into the flat gradient, and the fused Adam's first step
    equals torch.optim.Adam (eps 1e-15) on the unscaled gradient."""
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.trainer import NGPTrainer
    torch.manual_seed(0)
    m = VoxelGrid(grid_size=24, grid_radius=0.05, sh_degree=1).to(DEV)
    with torch.no_grad():
        m.sh_fields.uniform_(-1, 1)
        m.density_fields.uniform_(-0.5, 1)
    p0 = [p.detach().clone() for p in m.parameters()]
    tr = NGPTrainer(m, lr=1e-2, max_steps=100)
    assert tr.loss_scale == 2 ** 19 and m.grad_sink is not None
    x = (torch.rand(4000, 3, device=DEV) - 0.5)
    d = torch.randn(4000, 3, device=DEV)
    a, b = torch.randn(4000, device=DEV), torch.randn(4000, 3, device=DEV)
    sigma, rgb = m(x, d)
    ((sigma * a).sum() + (rgb * b).sum()).mul(tr.loss_scale).backward()
    grads = [p.grad.detach().clone() for p in m.parameters()]
    assert all(float(g.abs().max()) > 0 for g in grads)
    tr.optimizer_step()
    ref = [q.clone().requires_grad_(True) for q in p0]
    opt = torch.optim.Adam(ref, lr=1e-2, betas=(0.9, 0.999), eps=1e-15)
    for q, g in zip(ref, grads):
        q.grad = g / tr.loss_scale
    opt.step()
    for p, q in zip(m.parameters(), ref):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=2e-6, atol=1e-7)
    assert not any(bool(p.grad.any()) for p in m.parameters())     # the fused pass zeroes the gradient
    assert NGPTrainer(VoxelGrid(sh_degree=0, grid_size=4, half_opt=True).to(DEV)).loss_scale == 2 ** 16
    tr.detach()
    assert m.grad_sink is None


def _small_scene_model(steps):
    """A VoxelGrid trained for `steps` module-path steps on the 100x100 analytic scene."""
    from datasets.ray_utils import get_rays
    from modules.rendering import MAX_SAMPLES
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.trainer import NGPTrainer
    from test_gpu_e2e import _small_dataset
    torch.manual_seed(23)
    ds = _small_dataset(root_dir='', split='train', downsample=1.0, seed=23).to(DEV)
    ds.batch_size = 4096
    ds.ray_sampling_strategy = 'all_images'
    m = VoxelGrid().to(DEV)
    m.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    tr = NGPTrainer(m, lr=1e-2, max_steps=steps)
    for step in range(steps):
        data = ds[step % len(ds)]
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            if step % 16 == 0:
                m.update_density_grid(0.01 * MAX_SAMPLES / 3 ** 0.5, warmup=step < 256)
        o, dd = get_rays(data['direction'], data['pose'])
        tr.step(o, dd, data['rgb'])
    return m, ds


def test_render_test_time_matches_incremental_loop():
    """render(test_time=True) (one march per ray block + the module forward) against the reference's incremental
    loop: same samples, same fp32 model outputs; only the compositing's fp32 sums are grouped differently."""
    from datasets.ray_utils import get_rays
    from modules.intersection import ray_aabb_intersection
    from modules.rendering import _render_rays_test, render
    m, ds = _small_scene_model(200)
    m.eval()
    o, d = get_rays(ds.directions, ds.poses[0])
    with torch.no_grad(), torch.autocast('cuda', dtype=torch.float16):
        a = render(m, o, d, test_time=True)
        b = _render_rays_test(m, o.contiguous(), d.contiguous(), ray_aabb_intersection(o, d, m.scale))
    assert int(a['total_samples']) > 0
    for k in ('rgb', 'opacity'):
        torch.testing.assert_close(a[k].float(), b[k].float(), rtol=0, atol=1e-4)
    torch.testing.assert_close(a['depth'].float(), b['depth'].float(), rtol=1e-4, atol=1e-4)


def test_train_main_end_to_end_and_psnr(tmp_path, monkeypatch):
    """train.main with --model_name svox trains on the analytic scene, writes results/model.pth, which reloads into a
    VoxelGrid and through --ckpt_path; the test views reach the PSNR gate."""
    import train
    from modules.voxel_grid import VoxelGrid
    from test_gpu_e2e import _small_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _small_dataset})
    args = ['--dataset_name', 'synthetic', '--model_name', 'svox', '--batch_size', '4096']
    psnrs = train.main(args + ['--max_steps', '1000'])
    ckpt = tmp_path / 'results' / 'model.pth'
    assert ckpt.exists() and (tmp_path / 'results' / 'rgb_000.png').exists()
    sd = torch.load(ckpt, map_location='cpu')
    assert sd['sh_fields'].shape == (256, 256, 256, 27) and sd['density_fields'].shape == (256, 256, 256, 1)
    print("svox train.py psnr", psnrs)
    assert min(psnrs) > PSNR_GATE, psnrs
    m = VoxelGrid(**train.build_model_config(train.get_opts(args)))
    m.load_state_dict(sd)
    assert torch.equal(m.density_fields.detach(), sd['density_fields'])
    again = train.main(args + ['--max_steps', '1', '--ckpt_path', str(ckpt)])
    assert min(again) > 15.0, again


# Measured once after 1000 steps: views 18.4, 20.0, 20.8, 20.0 dB (mean 19.8) on an H100 80GB HBM3 at a 700 W power
# limit; an untrained model scores about 11 dB.  The gate is 2 dB below the worst view (the atomic sums make training
# slightly non-deterministic).
PSNR_GATE = 16.4
