"""--random_bg (DESIGN.md §6f): the per-ray colour draw against a numpy Philox4x32-10, the random-background head kernel
against fp64 (with and without alpha, with and without the distortion loss), the graph-captured step against the
module path, and train.py on a Blender-layout export of the teacher."""
import numpy as np
import pytest

import test_gpu_graph_step_distortion as tgd
from composite_ref import U  # noqa: F401  (the comparator's unit roundoff)

pytestmark = pytest.mark.gpu

M32 = 0xFFFFFFFF
BG_WORD = 0x62670001


def np_philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on uint64 arrays holding 32-bit words."""
    c = [np.asarray(x, np.uint64) & M32 for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0 & M32), np.uint64(k1 & M32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & np.uint64(M32), (p0 >> np.uint64(32)) ^ c[3] ^ k1,
             p0 & np.uint64(M32)]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & np.uint64(M32), (k1 + np.uint64(0xBB67AE85)) & np.uint64(M32)
    return c


def np_random_bg(seed, step, n):
    r = np.arange(n, dtype=np.uint64)
    v = np_philox(r, r >> np.uint64(32), np.full(n, step, np.uint64), np.full(n, BG_WORD, np.uint64), seed, seed >> 32)
    return np.stack([(x >> np.uint64(8)).astype(np.float32) * np.float32(5.9604644775390625e-8) for x in v[:3]], 1)


def test_draw_matches_numpy_philox():
    import torch
    from taichi_nerfs_b200 import ops
    for seed, step, n in ((23, 1, 1000), (24, 7, 333), ((1 << 40) + 5, 123456, 4097)):
        got = ops.random_bg(seed, step, n, 'cuda').cpu().numpy()
        assert np.array_equal(got, np_random_bg(seed, step, n)), (seed, step)
        assert got.min() >= 0 and got.max() < 1
        dev = ops.random_bg(seed, 0, n, 'cuda', step_dev=torch.tensor([step], device='cuda', dtype=torch.int32))
        assert np.array_equal(dev.cpu().numpy(), got)
    assert not np.array_equal(np_random_bg(23, 1, 64), np_random_bg(23, 2, 64))
    assert not np.array_equal(np_random_bg(23, 1, 64), np_random_bg(24, 1, 64))


# ---- the head kernel against fp64 ---------------------------------------------------------------------------------
def head_ref_rbg(sig, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, thr, n_active=None, faults=()):
    """tests/test_gpu_graph_step_distortion.py's head_ref with bg = (colours [n, 3], alpha [n] or None, b_load): the
    prediction composites onto the ray's colour, the target's loader background is swapped for it where alpha < 1, and
    dL/dopacity = -sum_c c_c g_c."""
    cols, alpha, b_load = bg
    n, S = rays_a.shape[0], sig.size
    z, zs = np.zeros(n), np.zeros(S)
    c = cols.astype(np.float64)
    fwd = tgd.np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, z, z, np.zeros((n, 3)), zs, n_active=n_active)
    out = fwd["rgb"] + c * (1 - fwd["op"])[:, None]
    tgt = gt.astype(np.float64)
    if alpha is not None:
        tgt = tgt + (c - b_load) * (1 - alpha.astype(np.float64))[:, None]
    dd = out - tgt
    g = scale * 2 * dd / (3 * n)
    go = -(c * g).sum(1)
    loss_ray, lmag, dw, gmag = tgd.np_distortion_f64(fwd["w"], deltas, ts, rays_a)
    gw = scale * w_d / n * dw
    ref = tgd.np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, z, g, gw, n_active=n_active)
    ref["mag"] = tgd.np_composite_f64(sig, rgbs, deltas, ts, rays_a, thr, go, z, g, scale * w_d / n * gmag,
                                      n_active=n_active)["mag"]
    loss = (dd ** 2).sum() + 3 * w_d * loss_ray.sum()
    return dict(fwd=fwd, out=out, dd=dd, ref=ref, loss=loss, loss_ray=loss_ray, lmag=lmag, gw=gw)


def _head_rbg(lib, t_in, cols, alpha, b_load, n, half, scale, thr, w_d):
    import torch
    from taichi_nerfs_b200 import _lib
    sig, rgbs, dl, ts, ra, gt = t_in
    S = sig.numel()
    loss_sum, op, rgb = torch.zeros(1, device='cuda'), torch.zeros(n, device='cuda'), torch.zeros(n, 3, device='cuda')
    dsig = torch.full((S,), 9.0, device='cuda')
    drgbs = torch.full((S, 3), 9.0, device='cuda', dtype=torch.float16 if half else torch.float32)
    P = tgd._P
    _lib.check(lib.ngp_ray_head_fused_random_bg(P(sig), P(rgbs), tgd.F16 if half else tgd.F32, P(dl), P(ts), P(ra),
                                                P(gt), P(cols), P(alpha), b_load, scale, None, thr, w_d, P(loss_sum),
                                                P(op), P(rgb), P(dsig), P(drgbs), n, tgd._ST()))
    return loss_sum, op, rgb, dsig, drgbs


@pytest.mark.parametrize("w_d", [0.0, 1e-2])
@pytest.mark.parametrize("with_alpha", [False, True])
@pytest.mark.parametrize("half", [False, True])
def test_random_bg_head_against_fp64(monkeypatch, half, with_alpha, w_d):
    from taichi_nerfs_b200 import _lib
    lib = _lib.load()
    sig, rgbs, deltas, ts, rays_a, gt = case = tgd._gpu_case(half, 0.0, 1e-4)
    n, scale, b_load = rays_a.shape[0], 2.0 ** 16, 1.0
    rng = np.random.default_rng(5)
    cols = np_random_bg(23, 4, n)
    alpha = rng.random(n).astype(np.float32) if with_alpha else None
    if with_alpha:
        alpha[:2] = (0.0, 1.0)
    got = _head_rbg(lib, [tgd._T(a) for a in case], tgd._T(cols), None if alpha is None else tgd._T(alpha), b_load,
                    n, half, scale, 1e-4, w_d)
    got = tuple(tgd._N(t) for t in got)
    monkeypatch.setattr(tgd, "head_ref", head_ref_rbg)
    tgd.check_head_dist(got, *case, (cols, alpha, b_load), scale, w_d, 1e-4, half,
                        f"half={half} alpha={with_alpha} w_d={w_d}")


@pytest.mark.parametrize("w_d", [0.0, 1e-2])
def test_random_bg_head_with_white_equals_constant_head(w_d):
    """Colours all 1 and no alpha: bit for bit the constant-background head with bg = 1."""
    import torch
    from taichi_nerfs_b200 import _lib
    lib = _lib.load()
    case = tgd._gpu_case(True, 0.0, 1e-4)
    t_in = [tgd._T(a) for a in case]
    n = case[4].shape[0]
    a = tgd._head(lib, t_in, n, True, 2.0 ** 16, 1e-4, w_d, plain=w_d == 0)
    b = _head_rbg(lib, t_in, torch.ones(n, 3, device='cuda'), None, 1.0, n, True, 2.0 ** 16, 1e-4, w_d)
    for x, y, name in zip(a[1:], b[1:], ("opacity", "rgb", "dsigma", "drgb")):
        assert torch.equal(x, y), name


# ---- the graph-captured step against the module path ----------------------------------------------------------------
@pytest.mark.parametrize("use_graph", [False, True])
def test_random_bg_graph_step_equals_module_path(lego_bitfield, monkeypatch, use_graph):
    """StaticTrainStep(random_bg=True).step(..., alpha) == NGPTrainer.step(bg_rgb=ops.random_bg(seed, s), alpha): the
    criteria of test_static_graph_step_with_distortion_equals_autograd_step; the step's colours are the numpy draw at
    the step's own counter, new at every step."""
    import torch
    from modules.networks import NGP
    from oracle.train_step import make_rays
    from taichi_nerfs_b200 import ops
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer

    def build():
        torch.manual_seed(3)
        m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
        with torch.no_grad():
            m.pos_encoder.hash_table.mul_(2e3)
            m.density_bitfield.copy_(torch.from_numpy(lego_bitfield))
        return m, NGPTrainer(m, lr=1e-2)

    n, seed = 2048, 29
    o, d = make_rays(n, seed=9)
    o, d = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    gt = torch.rand(n, 3, device='cuda')
    alpha = torch.rand(n, device='cuda')
    noise = torch.rand(n, device='cuda')

    m1, t1 = build()
    monkeypatch.setattr(torch, 'rand_like', lambda t, **k: noise.clone())
    losses1 = []
    for _ in range(3):
        cols = ops.random_bg(seed, t1.step_count + 1, n, 'cuda')
        losses1.append(float(t1.step(o, d, gt, bg_rgb=cols, alpha=alpha, b_load=1.0)[0]))
    monkeypatch.undo()

    m2, t2 = build()
    fs = StaticTrainStep(t2, n, samples_per_ray_capacity=64, use_graph=use_graph, random_bg=True, bg_seed=seed,
                         bg_load=1.0)
    losses2 = []
    for s in range(1, 4):
        losses2.append(float(fs.step(o, d, gt, noise=noise, alpha=alpha)))
        assert np.array_equal(fs.bg_rgb.cpu().numpy(), np_random_bg(seed, s, n)), s
    fs.flush()
    assert int(fs.counter[0]) > 1000
    for a, b in zip(losses1, losses2):
        assert abs(a - b) < 2e-3 * max(a, 1e-6), (losses1, losses2)
    for p1, p2 in zip(m1.parameters(), m2.parameters()):
        diff = (p1 - p2).abs()
        assert float((diff > 2e-3).float().mean()) < 2e-3, float(diff.max())
    assert t2.step_count == 3 and int(fs.bg_step) == 3
    # the per-ray colour reaches the loss: the same first step with another seed differs
    _, t3 = build()
    other = float(StaticTrainStep(t3, n, samples_per_ray_capacity=64, use_graph=use_graph, random_bg=True,
                                  bg_seed=seed + 1).step(o, d, gt, noise=noise, alpha=alpha))
    assert abs(other - losses2[0]) > 1e-3 * losses2[0]


def test_random_bg_refusals():
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200 import _lib
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    fs = StaticTrainStep(NGPTrainer(m), 256, samples_per_ray_capacity=8, use_graph=False, random_bg=True)
    with pytest.raises(_lib.NgpError, match='random_bg'):
        fs.attach_ray_source(torch.rand(2, 16, 3), torch.rand(2, 3, 4), torch.rand(16, 3))
    plain = StaticTrainStep(NGPTrainer(m), 256, samples_per_ray_capacity=8, use_graph=False)
    with pytest.raises(ValueError, match='alpha'):
        plain.step(torch.rand(256, 3, device='cuda'), torch.rand(256, 3, device='cuda'),
                   torch.rand(256, 3, device='cuda'), alpha=torch.ones(256, device='cuda'))


def test_train_random_bg_on_blender_export(tmp_path, monkeypatch, capsys):
    """train.py --dataset_name nerf --graph_step --random_bg on the RGBA teacher export: trains (reported beside the
    run without the flag in tests/test_gpu_disk_datasets.py)."""
    import train
    from test_gpu_disk_datasets import _export_blender, _teacher
    teacher = _teacher()
    root = str(tmp_path / 'lego_blender')
    _export_blender(root, teacher, 32, 2, 0.25)
    monkeypatch.chdir(tmp_path)
    psnrs = {}
    for extra in ([], ['--random_bg']):
        for path in ([], ['--graph_step']):
            p = train.main(['--dataset_name', 'nerf', '--root_dir', root, '--downsample', '0.25', '--half_opt',
                            '--max_steps', '1499'] + path + extra)
            psnrs[' '.join(path + extra) or 'module path'] = sum(p) / len(p)
    with capsys.disabled():
        print("\nblender layout, 1500 steps, held-out PSNR: " + "; ".join(f"{k}: {v:.2f} dB" for k, v in psnrs.items()))
    assert psnrs['--graph_step --random_bg'] > 25.0 and psnrs['--random_bg'] > 25.0
