"""Depth supervision (--depth_loss_w, DESIGN.md §6h) on the GPU:

- ngp_ray_head_fused_depth against the fp64 restatement (tests/depth_ref.py) and against the module path's kernels
  (composite_train_fwd -> torch loss -> composite_train_bwd(dL_ddepth)), fp16 / fp32 colours, every distortion x
  background combination; rays with and without targets (0, negative, NaN, inf), a ray that misses, a wall mid-chunk
  and a ray alive past 4096 samples;
- depth_w = 0 against the matching existing entry, bit for bit;
- StaticTrainStep(depth_loss_w) against NGPTrainer.step(extra_loss=depth_loss), hash fp16 and svox; its refusals;
- training on sparse views of the analytic scene with and without the depth loss: held-out depth error, PSNR and the
  Chamfer distance of the exported mesh; train.py on an ngp scene with 16-bit depth PNGs.

Every bound prints the value measured beside it (pytest -s)."""
import json
import os
import re

import numpy as np
import pytest

import test_gpu_graph_step_distortion as tgd
from composite_ref import U, kernel_termination
from depth_ref import check_head_depth, depth_valid

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _report(name, value):
    print(f"measured {name}: {value}")


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def _depth_targets(rays_a, seed):
    """Targets near each ray's own sample range, and rays without one: 0, negative, NaN and inf."""
    rng = np.random.default_rng(seed)
    n = rays_a.shape[0]
    d = rng.uniform(0.05, 2.0, n).astype(np.float32)
    ids = rays_a[:, 0]
    d[ids[[1, 3, 4, 8]]] = (0.0, -1.0, np.nan, np.inf)     # 1, 32, 33 and 12 samples: no target
    return d                                                 # the 0-sample ray (ids[0]) keeps a target: a miss


def _launch(lib, t_in, n, half, scale, thr, w_d, bgk, w_z, dgt, entry="depth"):
    """One head launch on outputs pre-filled with 9; bgk: None (constant 1) or (colours, alpha, b_load) tensors.
    entry: "depth" (ngp_ray_head_fused_depth) or "old" (the existing entry of that combination)."""
    import torch
    from taichi_nerfs_b200 import _lib
    sig, rgbs, dl, ts, ra, gt = t_in
    S = sig.numel()
    loss_sum, op, rgb = torch.zeros(1, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, 3, device=DEV)
    dsig = torch.full((S,), 9.0, device=DEV)
    drgbs = torch.full((S, 3), 9.0, device=DEV, dtype=torch.float16 if half else torch.float32)
    P, dt = tgd._P, tgd.F16 if half else tgd.F32
    cols, alpha, b_load = bgk if bgk is not None else (None, None, 1.0)
    if entry == "depth":
        _lib.check(lib.ngp_ray_head_fused_depth(P(sig), P(rgbs), dt, P(dl), P(ts), P(ra), P(gt), 1.0, P(cols), P(alpha),
                                                b_load, scale, None, thr, w_d, P(dgt), w_z, P(loss_sum), P(op), P(rgb),
                                                P(dsig), P(drgbs), n, tgd._ST()))
    elif bgk is not None:
        _lib.check(lib.ngp_ray_head_fused_random_bg(P(sig), P(rgbs), dt, P(dl), P(ts), P(ra), P(gt), P(cols), P(alpha),
                                                    b_load, scale, None, thr, w_d, P(loss_sum), P(op), P(rgb), P(dsig),
                                                    P(drgbs), n, tgd._ST()))
    else:
        return tgd._head(lib, t_in, n, half, scale, thr, w_d, plain=w_d == 0)
    return loss_sum, op, rgb, dsig, drgbs


def _module_chain(t_in, n, scale, thr, w_d, bgk, w_z, dgt):
    """The module path's kernels: composite_train_fwd -> the loss in torch (fp32) -> distortion_bwd ->
    composite_train_bwd with dL_ddepth = scale w_z 2 v (D - D^) / n."""
    import torch
    from modules.depth import depth_loss
    from taichi_nerfs_b200 import ops
    sig, rgbs, dl, ts, ra, gt = t_in
    _, op, dep, rgb, ws = ops.composite_train_fwd(sig, rgbs, dl, ts, ra, thr)
    if bgk is None:
        c, tgt = torch.ones(n, 3, device=DEV), gt
    else:
        c, alpha, b_load = bgk
        tgt = gt if alpha is None else gt + (c - b_load) * (1 - alpha)[:, None]
    out = rgb + c * (1 - op)[:, None]
    d = out - tgt
    g_rgb = scale * 2 * d / (3 * n)
    g_op = -(c * g_rgb).sum(1)
    dep_r = dep.clone().requires_grad_(True)
    lz = depth_loss({'depth': dep_r}, dgt)
    (scale * w_z * lz.mean()).backward()
    dist = ops.distortion_fwd(ws, dl, ts, ra)
    dws = ops.distortion_bwd(torch.full((n,), scale * w_d / n, device=DEV), ws, dl, ts, ra)
    dsig, drgbs = ops.composite_train_bwd(g_op, dep_r.grad.contiguous(), g_rgb, dws, sig, rgbs, dl, ts, ra, thr)
    loss = (d ** 2).sum() + 3 * w_d * dist.sum() + 3 * w_z * lz.detach().sum()
    return tuple(tgd._N(x) for x in (loss.reshape(1), op, out, dsig, drgbs))


@pytest.mark.parametrize("rbg", [False, True])
@pytest.mark.parametrize("w_d", [0.0, 1e-2])
@pytest.mark.parametrize("half", [False, True])
def test_depth_head_against_fp64_and_module_path(lib, half, w_d, rbg):
    import torch
    from test_gpu_random_bg import np_random_bg
    case = tgd._gpu_case(half, 0.0, 1e-4)
    sig, rgbs, deltas, ts, rays_a, gt = case
    n, scale, w_z, thr = rays_a.shape[0], 2.0 ** 16, 0.5, 1e-4
    dgt = _depth_targets(rays_a, 3 + half)
    t_in = [tgd._T(a) for a in case]
    if rbg:
        cols = np_random_bg(23, 4, n)
        alpha = np.random.default_rng(5).random(n).astype(np.float32)
        bg_np, bgk = (cols, alpha, 1.0), (tgd._T(cols), tgd._T(alpha), 1.0)
    else:
        bg_np, bgk = 1.0, None
    what = f"half={half} w_d={w_d} rbg={rbg}"
    got = tuple(tgd._N(t) for t in _launch(lib, t_in, n, half, scale, thr, w_d, bgk, w_z, tgd._T(dgt)))
    h, st = check_head_depth(got, *case, bg_np, scale, w_d, w_z, dgt, thr, half, what)
    _report(f"fused vs fp64 [{what}]", st)
    act = h["ref"]["active"]
    r6, r7 = rays_a[6], rays_a[7]
    assert act[r6[1]:r6[1] + r6[2]].all(), "the 5000-sample ray must stay alive past 4096 samples"
    assert not act[r7[1] + 4300], "the 4600-sample ray must stop at its wall"
    assert h["v"].sum() == n - 4 and h["dz"][rays_a[0, 0]] != 0
    # the depth term is visible at these bounds: the same output fails without it
    with pytest.raises(AssertionError):
        check_head_depth(got, *case, bg_np, scale, w_d, w_z, dgt, thr, half, "no gz", faults=("no_gz",))
    # the module path's kernels: within the fp64 bound too, and within twice it of the fused head
    chain = _module_chain(t_in, n, scale, thr, w_d, bgk, w_z, tgd._T(dgt))
    hc, stc = check_head_depth(chain, *case, bg_np, scale, w_d, w_z, dgt, thr, half, what + " module chain")
    _report(f"module chain vs fp64 [{what}]", stc)
    assert np.array_equal(kernel_termination(got[3], got[4], rays_a), kernel_termination(chain[3], chain[4], rays_a))
    ref = h["ref"]
    tol = 2 * 8 * ref["k"] * U * ref["mag"]
    e = np.abs(got[3].astype(np.float64) - chain[3])
    _report(f"fused vs module chain dsigma err / tol [{what}]", float((e / np.maximum(tol, 1e-300)).max()))
    assert (e <= tol).all(), "dsigma: fused vs module chain"
    assert np.abs(got[4].astype(np.float64) - chain[4]).max() <= (2 ** -10 if half else 1e-6) * np.abs(chain[4]).max()
    _report(f"loss fused / module chain [{what}]", (float(got[0][0]), float(chain[0][0])))
    assert abs(float(got[0][0]) - float(chain[0][0])) <= 1e-5 * abs(float(chain[0][0]))
    torch.cuda.synchronize()


@pytest.mark.parametrize("rbg", [False, True])
@pytest.mark.parametrize("w_d", [0.0, 1e-2])
@pytest.mark.parametrize("half", [False, True])
def test_depth_head_zero_weight_equals_existing_entry(lib, half, w_d, rbg):
    import torch
    case = tgd._gpu_case(half, 0.0, 1e-4)
    rays_a = case[4]
    n = rays_a.shape[0]
    t_in = [tgd._T(a) for a in case]
    bgk = None
    if rbg:
        rng = np.random.default_rng(9)
        bgk = (tgd._T(rng.random((n, 3)).astype(np.float32)), tgd._T(rng.random(n).astype(np.float32)), 1.0)
    dgt = tgd._T(_depth_targets(rays_a, 1))
    a = _launch(lib, t_in, n, half, 2.0 ** 16, 1e-4, w_d, bgk, 0.0, dgt)
    b = _launch(lib, t_in, n, half, 2.0 ** 16, 1e-4, w_d, bgk, 0.0, dgt, entry="old")
    for x, y, name in zip(a[1:], b[1:], ("opacity", "rgb", "dsigma", "drgb")):
        assert torch.equal(x, y), name
    # loss_sum: per-ray terms bit-identical, summed by atomics in an order that varies
    assert abs(float(a[0]) - float(b[0])) <= n * U * float(b[0])


def test_depth_head_device_loss_scale(lib):
    """scale_dev holding s == the host constant s, bit for bit (power-of-two scales)."""
    import torch
    from taichi_nerfs_b200 import _lib
    case = tgd._gpu_case(True, 0.0, 1e-4)
    t_in = [tgd._T(a) for a in case]
    sig, rgbs, dl, ts, ra, gt = t_in
    n, S = case[4].shape[0], case[0].size
    dgt = tgd._T(_depth_targets(case[4], 2))
    outs = []
    for s, dev in ((2.0 ** 16, None), (12345.0, torch.tensor([2.0 ** 16], device=DEV))):
        o = (torch.zeros(1, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, 3, device=DEV),
             torch.zeros(S, device=DEV), torch.zeros(S, 3, device=DEV, dtype=torch.float16))
        P = tgd._P
        _lib.check(lib.ngp_ray_head_fused_depth(P(sig), P(rgbs), tgd.F16, P(dl), P(ts), P(ra), P(gt), 1.0, None, None,
                                                1.0, s, P(dev), 1e-4, 1e-2, P(dgt), 0.5, *(P(x) for x in o), n,
                                                tgd._ST()))
        outs.append(o)
    for x, y in zip(outs[0][1:], outs[1][1:]):
        assert torch.equal(x, y)


# ---- the graph-captured step -----------------------------------------------------------------------------------------
W_Z = 0.5


def test_graph_step_with_depth_equals_module_path_hash(lego_bitfield, monkeypatch):
    """StaticTrainStep(depth_loss_w) == NGPTrainer.step(extra_loss=w * depth_loss(res, depth).mean()), hash fp16, three
    steps: the criteria of tests/test_gpu_graph_step_distortion.py::test_static_graph_step_with_distortion_equals_..."""
    import torch
    from modules.depth import depth_loss
    from modules.networks import NGP
    from oracle.train_step import make_rays
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer

    def build():
        torch.manual_seed(3)
        m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
        with torch.no_grad():
            m.pos_encoder.hash_table.mul_(2e3)
            m.density_bitfield.copy_(torch.from_numpy(lego_bitfield))
        return m, NGPTrainer(m, lr=1e-2)

    n = 2048
    o, d = make_rays(n, seed=9)
    o, d = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    gt = torch.rand(n, 3, device='cuda')
    noise = torch.rand(n, device='cuda')
    dgt = torch.rand(n, device='cuda') * 1.5 + 0.5
    dgt[::7] = 0.0
    dgt[3::11] = float('nan')

    def module(w, k):
        m, t = build()
        monkeypatch.setattr(torch, 'rand_like', lambda t, **kw: noise.clone())
        el = (lambda res: w * depth_loss(res, dgt).mean()) if w > 0 else None
        losses = [float(t.step(o, d, gt, extra_loss=el)[0]) for _ in range(k)]
        monkeypatch.undo()
        return m, t, losses

    def fused(w, k):
        m, t = build()
        fs = StaticTrainStep(t, n, samples_per_ray_capacity=64, use_graph=True, overlap_optimizer=True,
                             depth_loss_w=w)
        losses = [float(fs.step(o, d, gt, noise=noise, depth=dgt if w > 0 else None)) for _ in range(k)]
        fs.flush()
        assert int(fs.counter[0]) > 1000
        return m, t, losses

    m1, t1, l1 = module(W_Z, 3)
    m2, t2, l2 = fused(W_Z, 3)
    _report("hash step losses module / fused", (l1, l2))
    for a, b in zip(l1, l2):
        assert abs(a - b) < 2e-3 * max(a, 1e-6), (l1, l2)
    worst = 0.0
    for p1, p2 in zip(m1.parameters(), m2.parameters()):
        frac = float(((p1 - p2).abs() > 2e-3).float().mean())
        worst = max(worst, frac)
    _report("hash step fraction of parameters off by > 2e-3", worst)
    assert worst < 2e-3
    # the depth term of the first loss, fused against module (difference of first-step losses with and without it)
    lz_f = fused(W_Z, 1)[2][0] - fused(0.0, 1)[2][0]
    lz_m = module(W_Z, 1)[2][0] - module(0.0, 1)[2][0]
    _report("hash step depth term fused / module", (lz_f, lz_m))
    assert lz_m > 20 * (n + 8) * U * l1[0]
    assert abs(lz_f - lz_m) <= 0.02 * lz_m + (n + 8) * U * 4 * l1[0], (lz_f, lz_m)


def test_graph_step_with_depth_equals_module_path_svox(monkeypatch):
    """The voxel grid: gradients of one step against NGPTrainer.forward_backward, the bound of
    tests/test_gpu_voxel_graph_step.py::test_svox_graph_step_equals_module_path; and the depth term moves them."""
    import torch
    import test_gpu_voxel_graph_step as VG
    from modules.depth import depth_loss
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    o, d, gt, noise = VG._batch(0)
    n = o.shape[0]
    gen = torch.Generator(device=DEV).manual_seed(4)
    dgt = torch.rand(n, device=DEV, generator=gen) * 1.5 + 0.3
    dgt[::5] = 0.0

    def module(w):
        m, t, _ = VG._build()
        monkeypatch.setattr(torch, "rand_like", lambda t, **k: noise.clone())
        el = (lambda res: w * depth_loss(res, dgt).mean()) if w > 0 else None
        loss, _ = t.forward_backward(o, d, gt, extra_loss=el)
        monkeypatch.undo()
        torch.cuda.synchronize()
        return float(loss.detach()), t.flat_grad.detach().cpu().numpy().copy()

    l1, g1 = module(W_Z)
    _, g0 = module(0.0)
    m2, t2, bits = VG._build()
    fs = StaticTrainStep(t2, VG.N_RAYS, samples_per_ray_capacity=VG.CFG["spr"], T_threshold=VG.THR, use_graph=True,
                         overlap_optimizer=True, depth_loss_w=W_Z)
    l2 = float(fs.step(o, d, gt, noise=noise, depth=dgt))
    snap = VG._snap(fs, bits)
    fs.flush()
    g2 = snap["flat_grad"]
    e = np.abs(g2 - g1)
    scale = np.abs(g1).max()
    st = dict(loss=(l1, l2), max=float(e.max() / scale), p999=float(np.percentile(e[g1 != 0], 99.9) / scale),
              depth_term_max=float(np.abs(g1 - g0).max() / scale))
    _report("svox graph step vs module path with depth", st)
    assert abs(l1 - l2) <= 2e-3 * l1
    assert st["max"] <= VG.MODULE_MAX and st["p999"] <= VG.MODULE_P999, st
    assert st["depth_term_max"] > 100 * VG.MODULE_MAX


def test_graph_step_depth_refusals():
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200 import _lib
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    for w in (-1e-2, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            StaticTrainStep(NGPTrainer(m), 256, samples_per_ray_capacity=8, use_graph=False, depth_loss_w=w)
    fs = StaticTrainStep(NGPTrainer(m), 256, samples_per_ray_capacity=8, use_graph=False, depth_loss_w=0.1)
    z3, z1 = torch.zeros(256, 3, device=DEV), torch.zeros(256, device=DEV)
    with pytest.raises(ValueError, match="depth"):
        fs.step(z3, z3, z3)
    with pytest.raises(_lib.NgpError, match="depth"):
        fs.attach_ray_source(torch.zeros(2, 16, 3), torch.zeros(2, 3, 4), torch.zeros(16, 3))
    plain = StaticTrainStep(NGPTrainer(m), 256, samples_per_ray_capacity=8, use_graph=False)
    with pytest.raises(ValueError, match="depth"):
        plain.step(z3, z3, z3, depth=z1)
    torch.cuda.synchronize()


# ---- end to end --------------------------------------------------------------------------------------------------------
# Sparse views: 4 training views of the analytic scene (100 x 100), 1000 steps, --half_opt --graph_step, the same 4
# held-out views; depth_loss_w = 0.1 against 0.  Measured in two runs on one H100 80GB HBM3 (700 W power limit):
# held-out depth_mae 0.0604 / 0.0710 -> 0.0408 / 0.0407, psnr_avg 27.84 / 27.55 -> 30.38 / 30.34 dB, Chamfer distance of
# the N = 128 mesh 0.0189 / 0.0230 -> 0.0165 / 0.0163 (DESIGN.md §6h).  The bounds leave margin for run-to-run
# variation: depth_mae at most 0.85 of the arm without depth (measured 0.68 / 0.57), PSNR at most 1 dB below it
# (measured 2.5 / 2.8 dB above), the depth-supervised mesh within 3 lattice spacings (0.0236) of the analytic one.  The
# unsupervised arm's Chamfer distance varies too much between runs to bound; it is reported.
SPARSE_STEPS = 1000
SPARSE_W = 0.1


def _sparse_dataset(**kw):
    from datasets.synthetic import SyntheticLego
    kw = dict(kw)
    kw.update(img_wh=(100, 100), focal=138.9, n_images=4, with_depth=True, scene='analytic')
    return SyntheticLego(**kw)


def _eval_line(out):
    line = [ln for ln in out.splitlines() if ln.startswith("evaluation:")][-1]
    return {k: float(v) for k, v in re.findall(r"(\w+)=([-0-9.e+naif]+)", line)}


def test_sparse_views_depth_loss_improves_held_out_depth(tmp_path, monkeypatch, capsys):
    import mc_ref as M
    import torch
    import train
    from datasets.synthetic import analytic_scene
    from test_gpu_mesh import _chamfer
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _sparse_dataset})
    n_mc, tau = 128, 10.0
    x = M.grid_points(n_mc, 0.5)
    sigma, _ = analytic_scene(torch.from_numpy(np.stack(x, -1).reshape(-1, 3)).float())
    rv, _, _ = M.marching_cubes(sigma.numpy().reshape(n_mc, n_mc, n_mc), tau, 0.5)
    res = {}
    for w in (0.0, SPARSE_W):
        d = tmp_path / f"w{w}"
        d.mkdir()
        monkeypatch.chdir(d)
        train.main(['--dataset_name', 'synthetic', '--half_opt', '--graph_step', '--batch_size', '4096',
                    '--max_steps', str(SPARSE_STEPS), '--depth_loss_w', str(w), '--extract_mesh',
                    '--mesh_res', str(n_mc), '--mesh_threshold', str(tau)])
        ev = _eval_line(capsys.readouterr().out)
        v, _, _, f = M.read_ply(str(d / 'results' / 'mesh.ply'))
        ev['chamfer'] = _chamfer(v, rv) if len(f) else float('inf')
        res[w] = ev
    with capsys.disabled():
        _report("sparse views (4) held-out metrics by depth_loss_w", json.dumps(res))
    off, on = res[0.0], res[SPARSE_W]
    assert on['depth_mae'] < 0.85 * off['depth_mae'], res
    assert on['psnr_avg'] > off['psnr_avg'] - 1.0, res
    assert on['chamfer'] < 0.0236, res


def _write_ngp_scene(root, n_views=8, wh=100, focal=138.9, depth_scale=1e-4):
    """An instant-ngp scene of the analytic scene: RGB PNGs, 16-bit depth PNGs (z-depth / depth_scale), OpenGL-style
    transform matrices (the loader negates their y and z axes)."""
    import torch
    from PIL import Image
    from datasets.ray_utils import get_ray_directions, get_rays
    from datasets.synthetic import hemisphere_poses, render_teacher
    os.makedirs(os.path.join(root, 'images'))
    os.makedirs(os.path.join(root, 'depth'))
    K = torch.tensor([[focal, 0, wh / 2], [0, focal, wh / 2], [0, 0, 1]])
    dirs = get_ray_directions(wh, wh, K).to(DEV)
    frames = []
    for k, pose in enumerate(hemisphere_poses(n_views, 1.4, 31)):
        o, d = get_rays(dirs, pose.to(DEV))
        rgb, dep = render_teacher(o, d, return_depth=True)
        img = (rgb.clamp(0, 1).reshape(wh, wh, 3).cpu().numpy() * 255 + 0.5).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(root, 'images', f'{k}.png'))
        raw = np.round(dep.reshape(wh, wh).cpu().numpy() / depth_scale).astype(np.uint16)
        Image.fromarray(raw).save(os.path.join(root, 'depth', f'{k}.png'))
        m = np.eye(4)
        m[:3, :4] = pose.numpy()
        m[:3, 1:3] *= -1
        frames.append({'file_path': f'images/{k}.png', 'depth_path': f'depth/{k}.png', 'transform_matrix': m.tolist()})
    with open(os.path.join(root, 'transforms.json'), 'w') as f:
        json.dump({'w': wh, 'h': wh, 'fl_x': focal, 'fl_y': focal, 'integer_depth_scale': depth_scale,
                   'frames': frames}, f)


def test_train_py_on_ngp_scene_with_depth(tmp_path, monkeypatch, capsys):
    import train
    from datasets import dataset_dict
    root = str(tmp_path / 'scene')
    _write_ngp_scene(root)
    ds = dataset_dict['ngp'](root, 'train', 1.0)
    assert ds.depths.shape == (8, 100 * 100) and float(ds.depths.max()) > 0.5
    monkeypatch.chdir(tmp_path)
    psnrs = train.main(['--dataset_name', 'ngp', '--root_dir', root, '--half_opt', '--batch_size', '4096',
                        '--max_steps', '300', '--depth_loss_w', str(SPARSE_W)])
    ev = _eval_line(capsys.readouterr().out)
    with capsys.disabled():
        _report("train.py ngp scene with depth", ev)
    assert 'depth_mae' in ev and np.isfinite(ev['depth_mae']) and ev['depth_mae'] < 0.1, ev
    assert min(psnrs) > 20.0, psnrs
    # a scene without depth is refused
    with pytest.raises(ValueError, match="no depth"):
        train.main(['--dataset_name', 'ngp', '--root_dir', os.path.join(os.path.dirname(__file__), 'golden',
                    'datasets', 'ngp_scene'), '--max_steps', '1', '--depth_loss_w', '0.1'])


def test_module_depth_valid_matches_restatement():
    import torch
    from modules.depth import depth_valid as dv
    x = np.array([1.0, 0.0, -1.0, np.nan, np.inf, 1e-30], np.float32)
    assert np.array_equal(dv(torch.from_numpy(x)).numpy(), depth_valid(x))


def test_teacher_and_analytic_depth_targets():
    """The teacher's and the analytic scene's samples carry z-depth: in front of the camera, inside the range the scene
    box allows from the camera's distance, and 0 where the view sees only background."""
    import torch
    from datasets.synthetic import SyntheticLego
    from datasets.teacher import TeacherLego, teacher_dir
    assert teacher_dir() is not None, "build() stages the teacher model"
    far = 1.396 + 0.5 * 3 ** 0.5                                  # camera distance + the box's half-diagonal
    t = TeacherLego(n_images=2, img_wh=(64, 64), focal=88.9, batch_size=512, with_depth=True).to(DEV)
    s = t[0]
    assert torch.equal(s['depth'], t.depths[s['img_idxs'], s['pix_idxs']])
    tv = TeacherLego(n_images=2, img_wh=(64, 64), focal=88.9, with_depth=True, split='test').to(DEV)
    d = tv[1]['depth']
    assert d.shape == (64 * 64,) and bool((d >= 0).all()) and float(d.max()) < far
    hit = d > 0.3
    _report("teacher view: fraction of pixels with depth > 0.3", float(hit.float().mean()))
    assert 0.05 < float(hit.float().mean()) < 0.95
    a = SyntheticLego(n_images=2, img_wh=(64, 64), focal=88.9, batch_size=512, scene='analytic', with_depth=True,
                      split='test').to(DEV)
    da = a[0]['depth']
    assert bool((da >= 0).all()) and float(da.max()) < 1.4 + 0.5 * 3 ** 0.5
    assert not TeacherLego(n_images=2, img_wh=(8, 8), focal=11.1).to(DEV)[0].keys() & {'depth'}
