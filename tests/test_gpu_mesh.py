"""GPU checks of the mesh export (DESIGN.md §6g): the marching-cubes kernels against the numpy restatement (tests/
mc_ref.py), the lattice mask, every model kind against the analytic scene, the teacher Lego, and the command line."""
import filecmp
import shutil

import numpy as np
import pytest
import torch

import mc_ref as M

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _report(name, value):
    """Print a measured value behind one of the bounds below (shown by `pytest -s`); the tests write no files."""
    print(f"measured {name}: {value}")


def _gpu_mc(lat, tau, bound):
    from taichi_nerfs_b200 import ops
    v, n, f = ops.marching_cubes(torch.from_numpy(lat).to(DEV), tau, bound)
    return v.cpu().numpy(), n.cpu().numpy(), f.cpu().numpy()


def _compare(lat, tau, bound):
    v, n, f = _gpu_mc(lat, tau, bound)
    rv, rn, rf = M.marching_cubes(lat, tau, bound)
    assert v.shape == rv.shape and f.shape == rf.shape
    assert np.array_equal(f, rf)
    assert np.array_equal(v.view(np.uint32), rv.view(np.uint32))
    assert np.abs(n - rn).max(initial=0) <= 2e-6
    return v, n, f


def _through_fill(lat, tau, seed):
    """Send the field through the lattice-fill path with NaN, +-inf and exact-tau values planted: the filled lattice
    must hold 0 where sigma is not finite and the value elsewhere (every cell occupied)."""
    from taichi_nerfs_b200 import ops
    n = lat.shape[0]
    rng = np.random.default_rng(seed)
    sigma = lat.reshape(-1).copy()
    k = max(1, sigma.size // 50)
    pos = rng.choice(sigma.size, 4 * k, replace=False)
    sigma[pos[:k]] = np.nan
    sigma[pos[k:2 * k]] = np.inf
    sigma[pos[2 * k:3 * k]] = -np.inf
    sigma[pos[3 * k:]] = np.float32(tau)
    bits = torch.full((128 ** 3 // 8,), 255, dtype=torch.uint8, device=DEV)
    out = torch.empty(n, n, n, device=DEV)
    chunk = max(1, sigma.size // 3 + 1)       # several chunks, as density_lattice runs them
    for start in range(0, sigma.size, chunk):
        cnt = min(chunk, sigma.size - start)
        _, occ = ops.mesh_lattice_points(n, 0.5, start, cnt, bits, 1, 128, 0.5)
        ops.mesh_lattice_store(torch.from_numpy(sigma[start:start + cnt]).to(DEV), occ, start, out)
    want = np.where(np.isfinite(sigma), sigma, np.float32(0)).reshape(n, n, n)
    got = out.cpu().numpy()
    assert np.array_equal(got, want)
    return got


@pytest.mark.parametrize("n", [2, 17, 64, 129, 300])
def test_random_fields_match_restatement(n):
    tau = 0.25
    lat = M.random_field(n, seed=n, threshold=tau, block=1 if n <= 129 else 7) if n > 2 else \
        np.random.default_rng(1).uniform(-1, 1, (2, 2, 2)).astype(np.float32)
    lat = _through_fill(lat, tau, seed=n)
    v, n_, f = _compare(lat, tau, 0.5)
    if n > 2:
        assert len(f) > 0 and M.is_closed_oriented(f)
    v2, n2, f2 = _gpu_mc(lat, tau, 0.5)
    assert np.array_equal(v, v2) and np.array_equal(n_, n2) and np.array_equal(f, f2)


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_analytic_fields_match_restatement(shape):
    lat = M.sphere_field(256, 0.5, 0.3) if shape == "sphere" else M.torus_field(256, 0.5, 0.25, 0.1)
    lat = _through_fill(lat, 0.0, seed=3)
    v, _, f = _compare(lat, 0.0, 0.5)
    # planted NaN / inf became 0 = tau: outside, so they punch small holes; the surface is still oriented
    _, dcount = M.edge_incidence(f)
    assert np.all(dcount == 1)


def test_clean_sphere_is_closed_and_repeatable():
    lat = M.sphere_field(256, 0.5, 0.3)
    v, n, f = _compare(lat, 0.0, 0.5)
    assert M.is_closed_oriented(f) and M.euler_characteristic(len(v), f) == 2
    vol = 4 / 3 * np.pi * 0.3 ** 3
    assert abs(M.signed_volume(v, f) - vol) < 0.01 * vol


def test_threshold_above_maximum_is_empty():
    lat = M.sphere_field(64, 0.5, 0.3)
    v, n, f = _gpu_mc(lat, float(lat.max()) + 1.0, 0.5)
    assert v.shape == (0, 3) and n.shape == (0, 3) and f.shape == (0, 3)


# ---- the occupancy mask --------------------------------------------------------------------------------------------
def _frexp_bit(x):
    m, e = np.frexp(x)
    return np.where(x == 0, 0, np.where(m == 0.5, e - 1, e))


def _morton(x, y, z):
    out = np.zeros_like(x, dtype=np.uint64)
    for b in range(10):
        for k, c in enumerate((x, y, z)):
            out |= ((c.astype(np.uint64) >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + k)
    return out


def _occupied_ref(xyz, bits, cascades, grid_size, scale):
    """The marcher's position rule restated in numpy fp32."""
    f32 = np.float32
    mx = np.abs(xyz).max(axis=1)
    mip = np.zeros(len(xyz), np.int64) if cascades == 1 else \
        np.minimum(cascades - 1, np.maximum(0, _frexp_bit(mx) + 1))
    mb = np.minimum(np.exp2(mip - 1.0).astype(f32), f32(scale))
    inv = f32(1) / mb
    g = f32(grid_size)
    v = (f32(0.5) * (xyz * inv[:, None] + f32(1))) * g
    u = np.clip(v, f32(0), g - f32(1)).astype(np.int64)
    idx = mip.astype(np.uint64) * np.uint64(grid_size ** 3) + _morton(u[:, 0], u[:, 1], u[:, 2])
    return (bits[(idx >> np.uint64(3)).astype(np.int64)] >> (idx & np.uint64(7)).astype(np.uint8)) & 1


@pytest.mark.parametrize("scale,n", [(0.5, 67), (2.0, 61), (8.0, 33)])
def test_lattice_mask_follows_marcher_rule(scale, n):
    from taichi_nerfs_b200 import ops
    cascades = max(1 + int(np.ceil(np.log2(2 * scale))), 1)
    rng = np.random.default_rng(n)
    bits = rng.integers(0, 256, cascades * 128 ** 3 // 8, dtype=np.uint8)
    xyz, occ = ops.mesh_lattice_points(n, scale, 0, n ** 3, torch.from_numpy(bits).to(DEV), cascades, 128, scale)
    xyz = xyz.cpu().numpy()
    x = M.node_coords(n, scale)
    gx, gy, gz = np.meshgrid(x, x, x, indexing="ij")
    assert np.array_equal(xyz, np.stack([gx, gy, gz], -1).reshape(-1, 3))
    assert np.array_equal(occ.cpu().numpy(), _occupied_ref(xyz, bits, cascades, 128, scale).astype(np.uint8))


def test_cleared_half_has_no_geometry():
    """With the cells of x < 0 cleared from a model's bitfield, the lattice is 0 there and no vertex lies in that
    half beyond the edges that leave its last node."""
    from modules.networks import NGP
    from taichi_nerfs_b200 import ops
    from taichi_nerfs_b200.mesh import density_lattice
    model = NGP(scale=0.5, max_res=1024).to(DEV).eval()
    coords = torch.stack(torch.meshgrid(*[torch.arange(128)] * 3, indexing="ij"), -1).reshape(-1, 3).int().to(DEV)
    idx = ops.morton3d(coords).long()
    bits = torch.zeros(128 ** 3, dtype=torch.bool, device=DEV)
    bits[idx[coords[:, 0] >= 64]] = True
    packed = (bits.view(-1, 8).to(torch.uint8) << torch.arange(8, device=DEV, dtype=torch.uint8)).sum(1)
    model.density_bitfield.copy_(packed.to(torch.uint8))
    sphere = lambda p: (40.0 * (0.3 - p.norm(dim=1))).exp()            # noqa: E731
    model._density_eval = lambda p: sphere(p)                           # an analytic density through the same path
    n = 96
    lat = density_lattice(model, n)
    x = torch.from_numpy(M.node_coords(n, 0.5)).to(DEV)
    assert torch.all(lat[x < 0] == 0) and torch.any(lat[x > 0] > 10.0)
    v, _, f = ops.marching_cubes(lat, 10.0, 0.5)
    assert len(f) > 0
    last_cleared = x[x < 0].max()
    assert torch.all(v[:, 0] > last_cleared)


# ---- every model kind against the analytic scene ------------------------------------------------------------------
def _small_dataset(**kw):
    from datasets.synthetic import SyntheticLego
    kw = dict(kw)
    kw.update(img_wh=(100, 100), focal=138.9, n_images=kw.get('n_images', 40))
    return SyntheticLego(**kw)


KINDS = {
    "hash_fp32": [],
    "hash_half": ["--half_opt"],
    "triplane": ["--encoder_type", "triplane"],
    "svox": ["--model_name", "svox"],
    "deployment": ["--deployment"],
}
# the voxel grid starts from a uniform density of 0.1 and grows it slowly: after 1500 steps its densest node held 4.4
# (H100 run), so it is meshed at tau = 2, and so is the analytic reference it is compared with
STEPS = {k: 1500 if k == "svox" else 300 for k in KINDS}
TAU = {k: 2.0 if k == "svox" else 10.0 for k in KINDS}
# mean symmetric Chamfer distance and mean colour error at N = 128 (spacing 1/127 = 0.0079), bound = measured + margin;
# measured on one H100 80GB HBM3 (700 W power limit): hash_fp32 0.0153 / 0.080, hash_half 0.0059 / 0.031,
# triplane 0.0187 / 0.124, deployment 0.0122 / 0.073, svox (tau = 2, 1500 steps) 0.0208 / 0.235.  Every Chamfer bound
# stays under 3 spacings (0.0236).
CHAMFER_BOUND = {"hash_fp32": 0.020, "hash_half": 0.010, "triplane": 0.023, "deployment": 0.016, "svox": 0.0235}
COLOR_BOUND = {"hash_fp32": 0.11, "hash_half": 0.05, "triplane": 0.16, "deployment": 0.10, "svox": 0.27}


def _chamfer(a, b):
    a, b = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)

    def one_way(p, q):
        return torch.cat([torch.cdist(p[i:i + 2048], q).min(1).values for i in range(0, len(p), 2048)]).double().mean()

    return float(0.5 * (one_way(a, b) + one_way(b, a)))


@pytest.mark.parametrize("kind", list(KINDS))
def test_model_kinds_mesh_the_analytic_scene(tmp_path, monkeypatch, kind):
    """train.py --extract_mesh on the analytic scene, then extract_mesh.py from the checkpoint: the same bytes, a mesh
    near the analytic scene's own, coloured like it."""
    import extract_mesh
    import train
    from datasets.synthetic import analytic_scene
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _small_dataset})
    n, tau = 128, TAU[kind]
    flags = ['--dataset_name', 'synthetic', '--batch_size', '4096'] + KINDS[kind] + \
        ['--mesh_res', str(n), '--mesh_threshold', str(tau)]
    train.main(flags + ['--max_steps', str(STEPS[kind]), '--extract_mesh'])
    ply = tmp_path / 'results' / 'mesh.ply'
    shutil.copy(ply, tmp_path / 'train_mesh.ply')
    extract_mesh.main(flags + ['--ckpt_path', str(tmp_path / 'results' / 'model.pth')])
    assert filecmp.cmp(ply, tmp_path / 'train_mesh.ply', shallow=False)

    v, nrm, col, f = M.read_ply(str(ply))
    assert len(f) > 0 and np.all(np.abs(v) <= 0.5)
    x = M.grid_points(n, 0.5)
    pts = torch.from_numpy(np.stack(x, -1).reshape(-1, 3)).float()
    sigma, _ = analytic_scene(pts)
    rv, _, rf = M.marching_cubes(sigma.numpy().reshape(n, n, n), tau, 0.5)
    cd = _chamfer(v, rv)
    _, rgb = analytic_scene(torch.from_numpy(v).double())
    mae = float(np.abs(col / 255.0 - rgb.numpy()).mean())
    _report(f"{kind}_chamfer", cd)
    _report(f"{kind}_color_mae", mae)
    assert cd < CHAMFER_BOUND[kind], cd
    assert mae < COLOR_BOUND[kind], mae


# ---- the teacher Lego -------------------------------------------------------------------------------------------
def test_teacher_lego_mesh_projects_onto_opaque_pixels():
    import __graft_entry__ as g
    if not g.stage_lego_fixture():
        pytest.skip("shipped Lego weights could not be staged")
    from datasets.ray_utils import get_ray_directions, get_rays
    from datasets.synthetic import hemisphere_poses
    from datasets.teacher import load_teacher
    from modules.rendering import render
    from taichi_nerfs_b200.mesh import extract_mesh
    model = load_teacher(DEV)
    mesh = extract_mesh(model, 256, 10.0)
    v = mesh.vertices
    assert len(v) > 0 and len(mesh.faces) > 0
    assert torch.all(v.abs() <= 0.5)
    assert torch.all((mesh.colors >= 0) & (mesh.colors <= 1))
    w = h = 400
    f = 1111.111 * w / 800
    K = torch.tensor([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]], dtype=torch.float32)
    dirs = get_ray_directions(h, w, K).to(DEV)
    fractions = []
    for pose in hemisphere_poses(2, 1.396, seed=1023).to(DEV):
        o, d = get_rays(dirs, pose)
        with torch.no_grad(), torch.autocast('cuda', dtype=torch.float16):
            res = render(model, o, d, test_time=True, exp_step_factor=0.0)
        opacity = res['opacity'].float().reshape(h, w)
        pc = (v - pose[:, 3]) @ pose[:, :3]                 # camera frame [right, down, front]
        u = torch.floor(pc[:, 0] / pc[:, 2] * f + w / 2).long()
        r = torch.floor(pc[:, 1] / pc[:, 2] * f + h / 2).long()
        ok = (pc[:, 2] > 0) & (u >= 0) & (u < w) & (r >= 0) & (r < h)
        hit = torch.zeros_like(ok)
        hit[ok] = opacity[r[ok], u[ok]] > 0.5
        fractions.append(float(hit.float().mean()))
    _report("lego_opaque_fraction", fractions)
    # measured 0.979 and 0.981 on one H100 80GB HBM3 (700 W power limit); what the other ~2 % are is not established
    # (candidates: faint fringes at tau = 10 that composite below 0.5 opacity, silhouette pixels)
    assert min(fractions) >= 0.97, fractions
