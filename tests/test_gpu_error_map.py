"""Error-map ray sampling on the GPU (DESIGN.md §6j): the four kernels against the integer restatement
(tests/error_map_ref.py) and torch, the graph-captured step with the map against the step without it, every model kind,
and the behaviour on the teacher Lego.

- sampler: img / pix / w bit for bit at n in {1, 255, 256, 257, 8192, 2^20}, T from 1 to 4.1 M tiles, W and H not
  multiples of R; a chi-square of 2^22 draws of a small skewed map (fixed seed, so the statistic is deterministic);
- accumulate: acc and cnt exactly, with the random-background target and clamped indices;
- rebuild: EMA, cleared counters, CDF and the workspace's (max E, S, M, status, k, c) exactly, and the shift that keeps
  M below 2^53;
- gradient weight: bit for bit against torch in fp32 and fp16, w = 1 the identity, rays with no samples, found_inf;
- graph step with a uniform map: bitwise wherever the step is deterministic, the loss and the table gradient within
  the reordering bounds of their atomic sums (as tests/test_gpu_extrinsics.py); the kernel counts;
- skewed map: the graph step's gradient against the module path's;
- teacher Lego: the share of drawn rays that see the object after 500 steps, and the held-out PSNR after 3000 steps.
Every bound prints the value measured beside it (pytest -s)."""
import numpy as np
import pytest

import error_map_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24


def _report(name, value):
    print(f"measured {name}: {value}")


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def _map(geom, E=None, seed=0):
    import torch
    from taichi_nerfs_b200.error_map import ErrorMap
    n_img, W, H, res = geom
    em = ErrorMap(n_img, W, H, res=res, seed=seed)
    if E is not None:
        em.E.copy_(torch.from_numpy(E))
        em.rebuild()   # no counts: E is kept, the CDF follows it
    return em


def _skewed_E(T, rng, hot=0.01):
    E = rng.integers(0, 1 << 22, T).astype(np.int64)
    idx = rng.choice(T, max(1, int(T * hot)), replace=False)
    E[idx] = rng.integers(1 << 29, 3 << 30, idx.size)
    return E


# ---- kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", [(1, 1, 1, 1), (3, 100, 75, 64), (2, 37, 53, 7), (1000, 100, 75, 64)])
def test_sampler_bit_exact(lib, geom):
    import torch
    rng = np.random.default_rng(geom[0] + geom[1])
    em = _map(geom, _skewed_E(geom[0] * geom[3] ** 2, rng), seed=0x1234_5678_9ABC)
    E, cdf, info = R.rebuild(em.E.cpu().numpy(), np.zeros(em.T, np.int64), np.zeros(em.T, np.int64), em.geom)
    assert np.array_equal(em.cdf.cpu().numpy(), cdf)
    ws = em.workspace.cpu().numpy()
    assert ws[[1, 2, 3, 4, 5]].tolist() == [info["S"], info["M"], 0, info["k"], info["c"]]
    for n in (1, 255, 256, 257, 8192, 1 << 20):
        step = n * 7 + 3
        img, pix, w = em.draw(n, step)
        ri, rp, rw = R.sample(cdf, em.geom, em.seed, step, n)
        assert np.array_equal(img.cpu().numpy(), ri) and np.array_equal(pix.cpu().numpy(), rp), n
        assert np.array_equal(w.cpu().numpy().view(np.uint32), rw.view(np.uint32)), n
        assert float(w.max()) <= em.max_weight
    # the step from device memory draws the same batch
    sd = torch.tensor([12345], device=DEV, dtype=torch.int32)
    a, b = em.draw(4096, 12345), em.draw(4096, 0, step_dev=sd)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_uniform_map_draws_weight_one(lib):
    em = _map((5, 123, 77, 64))
    _, _, w = em.draw(1 << 16, 9)
    assert bool((w == 1.0).all())


def test_sampler_chi_square(lib):
    from scipy.stats import chi2
    geom = (2, 9, 7, 3)
    E = np.array([0, 1, 5, 3 << 30, 2, 7, 1 << 28, 0, 9] * 2, np.int64)
    em = _map(geom, E, seed=99)
    n = 1 << 22
    img, pix, _ = em.draw(n, 1)
    t = R.tile_of(img.cpu().numpy(), pix.cpu().numpy(), geom)
    cdf = em.cdf.cpu().numpy()
    p = np.diff(np.concatenate([[0], cdf])) / cdf[-1]
    obs = np.bincount(t, minlength=em.T)
    stat = float(((obs - n * p) ** 2 / (n * p)).sum())
    pval = float(chi2.sf(stat, em.T - 1))
    _report("chi-square of 2^22 draws over 18 tiles (statistic, p-value)", (stat, pval))
    assert pval > 1e-3
    # inside a tile the pixel is uniform too: the tile with the largest mass, per pixel
    pix_np, img_np = pix.cpu().numpy(), img.cpu().numpy()
    big = int(np.argmax(p))
    sel = pix_np[(t == big) & (img_np == big // 9)]
    cnt = np.bincount(sel, minlength=63)
    cnt = cnt[cnt > 0]
    assert len(cnt) == R.tile_pixels(geom)[big]
    stat2 = float(((cnt - cnt.mean()) ** 2 / cnt.mean()).sum())
    assert chi2.sf(stat2, len(cnt) - 1) > 1e-3


@pytest.mark.parametrize("rbg", [False, True])
def test_accumulate_exact(lib, rbg):
    import torch
    geom = (4, 50, 30, 16)
    em = _map(geom)
    rng = np.random.default_rng(5 + rbg)
    n = 20000
    pred = rng.random((n, 3)).astype(np.float32) * 1.5
    tgt = rng.random((n, 3)).astype(np.float32)
    pred[:10] = np.nan
    img = rng.integers(-2, 6, n)       # some out of range: clamped
    pix = rng.integers(-5, 50 * 30 + 5, n)
    kw = {}
    if rbg:
        kw = dict(bg_rgb=rng.random((n, 3)).astype(np.float32), alpha=rng.random(n).astype(np.float32), b_load=1.0)
    acc, cnt = np.zeros(em.T, np.int64), np.zeros(em.T, np.int64)
    R.accumulate(acc, cnt, pred, tgt, img, pix, em.geom, **kw)
    T_ = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    tkw = {k: (T_(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    em.accumulate(T_(pred), T_(tgt), T_(img), T_(pix), **tkw)
    assert np.array_equal(em.acc.cpu().numpy(), acc) and np.array_equal(em.cnt.cpu().numpy(), cnt)
    assert acc.sum() > 0 and cnt.sum() == n


def test_rebuild_exact(lib):
    import torch
    geom = (7, 90, 61, 32)
    rng = np.random.default_rng(8)
    em = _map(geom, _skewed_E(7 * 32 * 32, rng))
    E0 = em.E.cpu().numpy()
    cnt = rng.integers(0, 5, em.T).astype(np.int64)      # tiles with cnt = 0 keep their E
    acc = rng.integers(0, 3 << 30, em.T).astype(np.int64) * cnt
    em.acc.copy_(torch.from_numpy(acc))
    em.cnt.copy_(torch.from_numpy(cnt.astype(np.int32)))
    em.rebuild()
    E, cdf, info = R.rebuild(E0, acc.copy(), cnt.copy(), em.geom)
    assert np.array_equal(em.E.cpu().numpy(), E) and np.array_equal(em.cdf.cpu().numpy(), cdf)
    assert not bool(em.acc.any()) and not bool(em.cnt.any())
    ws = em.workspace.cpu().numpy()
    assert ws[:6].tolist() == [info["emax"], info["S"], info["M"], 0, info["k"], info["c"]]
    img = torch.as_tensor(em.as_image())
    assert img.shape == (7, 32, 32) and torch.equal(img.flatten(), (em.E.double() / (1 << 30)).float())


def test_rebuild_shift_guards_the_cdf(lib):
    geom = (64, 4096, 4096, 64)   # N_pix = 2^30: the largest errors need k > 0 for M < 2^53
    rng = np.random.default_rng(2)
    E = np.full(64 * 64 * 64, 3 << 30, np.int64)
    E[rng.integers(0, E.size, 1000)] = 0
    em = _map(geom, E)
    _, cdf, info = R.rebuild(E, np.zeros(E.size, np.int64), np.zeros(E.size, np.int64), em.geom)
    ws = em.workspace.cpu().numpy()
    _report("shift k, M / 2^53", (info["k"], info["M"] / 2 ** 53))
    assert info["k"] > 0 and ws[4] == info["k"] and ws[3] == 0
    assert np.array_equal(em.cdf.cpu().numpy(), cdf) and cdf[-1] < 2 ** 53


def _rays_a(rng, n, S):
    """(ray, start, count) rows in shuffled order over S sample rows: some rays with 0 samples, one row past S."""
    counts = rng.integers(0, 12, n)
    counts[rng.integers(0, n, n // 10)] = 0
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    order = rng.permutation(n)
    ra = np.stack([order, starts[order], counts[order]], 1).astype(np.int32)
    return ra, int(counts.sum())


@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_grad_weight_bit_exact(lib, dtype):
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(3)
    n = 5000
    ra_np, S = _rays_a(rng, n, 0)
    dt = getattr(torch, dtype)
    ra = torch.from_numpy(ra_np).to(DEV)
    w = torch.from_numpy(rng.random(n).astype(np.float32) * 5).to(DEV)
    dsig = torch.randn(S, device=DEV)
    drgb = torch.randn(S, 3, device=DEV).to(dt)
    # reference: every row of ray r times w[r], one rounding
    row_ray = torch.empty(S, dtype=torch.long, device=DEV)
    for r, s, c in ra_np.tolist():
        row_ray[s:s + c] = r
    ws = w[row_ray]
    ref_s = dsig * ws
    ref_c = (drgb.float() * ws[:, None]).to(dt)
    a, b = dsig.clone(), drgb.clone()
    fi = torch.zeros(1, device=DEV, dtype=torch.int32)
    ops.ray_grad_weight(ra, w, a, b, found_inf=fi)
    assert torch.equal(a, ref_s) and torch.equal(b, ref_c) and int(fi) == 0
    # w = 1: the identity bit for bit
    a, b = dsig.clone(), drgb.clone()
    ops.ray_grad_weight(ra, torch.ones_like(w), a, b, found_inf=fi)
    assert torch.equal(a.view(torch.int32), dsig.view(torch.int32)) and torch.equal(b, drgb) and int(fi) == 0
    # n_rows clips the last rows: they stay as they were
    a, b = dsig.clone(), drgb.clone()
    ops.ray_grad_weight(ra, w, a, b, n_rows=S - 7)
    assert torch.equal(a[:S - 7], ref_s[:S - 7]) and torch.equal(a[S - 7:], dsig[S - 7:])
    # a non-finite result raises found_inf: an inf input, and (fp16) an overflow of a finite product
    a, b = dsig.clone(), drgb.clone()
    a[row_ray == int(ra_np[ra_np[:, 2] > 0][0, 0])] = float("inf")
    ops.ray_grad_weight(ra, w, a, b, found_inf=fi)
    assert int(fi) == 1
    if dtype == "float16":
        fi.zero_()
        b = torch.full_like(drgb, 60000.0)
        ops.ray_grad_weight(ra, torch.full_like(w, 2.0), dsig.clone(), b, found_inf=fi)
        assert int(fi) == 1 and bool(torch.isinf(b).any())


# ---- the training step ---------------------------------------------------------------------------------------------
def _batch(n, seed, n_img=6, wh=64):
    import torch
    from datasets.synthetic import SyntheticLego
    ds = SyntheticLego(n_images=n_img, img_wh=(wh, wh), focal=88.9, scene='random', with_rgb=False)
    g = torch.Generator().manual_seed(seed)
    pix = torch.randint(0, wh * wh, (n,), generator=g)
    img = torch.randint(0, n_img, (n,), generator=g)
    from datasets.ray_utils import get_rays
    o, d = get_rays(ds.directions[pix], ds.poses[img])
    return (o.to(DEV).contiguous(), d.to(DEV).contiguous(), img.to(DEV), pix.to(DEV),
            torch.rand(n, 3, generator=g).to(DEV), torch.rand(n, generator=g).to(DEV))


def _model(lego_bitfield):
    import torch
    from modules.networks import NGP
    torch.manual_seed(3)
    m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    with torch.no_grad():
        m.pos_encoder.hash_table.mul_(2e3)
        m.density_bitfield.copy_(torch.from_numpy(lego_bitfield))
    return m


def _graph_stages(lego_bitfield, batch, em, w=None):
    """One step's stages enqueued eagerly (no update).  Returns every per-ray buffer, the per-sample buffers in ray
    order, the loss, the inf flag, the table gradient and sum |term| of its scatter, and S."""
    import ctypes as C
    import torch
    from taichi_nerfs_b200._lib import load
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    o, d, img, pix, gt, noise = batch
    n = o.shape[0]
    t = NGPTrainer(_model(lego_bitfield), lr=1e-2)
    fs = StaticTrainStep(t, n, samples_per_ray_capacity=128, use_graph=False, error_map=em)
    for k, v in (("rays_o", o), ("rays_d", d), ("gt", gt), ("noise", noise)):
        getattr(fs, k).copy_(v)
    if em is not None:
        fs.em_img.copy_(img)
        fs.em_pix.copy_(pix)
        fs.ray_w.copy_(w)
    fs.counter.zero_()
    fs.loss_sum.zero_()
    t.found_inf.zero_()
    fs._enqueue_march()
    fs._enqueue_network()
    torch.cuda.synchronize()
    ra = fs.rays_a.long()
    counts = ra[:, 2]
    S = int(counts.sum())
    assert S == int(fs.counter[0]) and int(fs.counter[1]) == 0
    first = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    rows = torch.repeat_interleave(ra[:, 1], counts) + torch.arange(S, device=DEV) - first
    out = {k: getattr(fs, k).clone() for k in ("rays_o", "rays_d", "rgb", "opacity")}
    out["counts"] = counts.clone()
    for k in ("xyzs", "dirs", "ts", "deltas", "sig", "rgbs", "dsig", "drgbs", "demb"):
        out[k] = getattr(fs, k)[rows].clone()
    P = fs.P
    mag = torch.zeros_like(t.flat_grad)
    demb_abs = fs.demb.abs()
    rc = fs.enc.enqueue_encode_bwd_dyn(load(), C.c_void_p(fs.xyzs.data_ptr()), C.c_void_p(fs._table().data_ptr()),
                                       C.c_void_p(demb_abs.data_ptr()), C.c_void_p(mag.data_ptr()), fs.cap,
                                       C.c_void_p(fs.counter.data_ptr()), fs.aabb6, None,
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    return out, float(fs.loss_sum), int(t.found_inf), t.flat_grad.clone(), mag[:P], S, P


def test_graph_step_with_uniform_map_is_unchanged(lego_bitfield):
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    n = 4096
    batch = _batch(n, 4)
    em = _map((6, 64, 64, 64))
    _, _, w = em.draw(n, 0)
    assert bool((w == 1).all())
    on, l_on, f_on, g_on, mag, S, P = _graph_stages(lego_bitfield, batch, em, w)
    off, l_off, f_off, g_off, _, S_off, _ = _graph_stages(lego_bitfield, batch, None)
    assert S == S_off and S > 20000 and f_on == f_off == 0
    for k in on:
        assert torch.equal(on[k], off[k]), k
    dg = (g_on[:P] - g_off[:P]).abs()
    _report("graph step: loss on / off, max table-gradient difference / (2 S u sum|term|)",
            (l_on, l_off, float((dg / (2 * S * U * mag).clamp_min(1e-38)).max())))
    assert abs(l_on - l_off) <= 2 * n * U * l_off
    assert bool((dg <= 2 * S * U * mag).all()) and float(g_on[:P].abs().max()) > 0
    assert int(em.cnt.sum()) == n and int(em.acc.sum()) > 0    # the step's errors reached the map

    # graph replays: the host-fed step gains the accumulate and weight nodes, the sampled step also the sampler
    o, d, img, pix, gt, noise = batch
    t = NGPTrainer(_model(lego_bitfield), lr=1e-2)
    em2 = _map((6, 64, 64, 64))
    fs = StaticTrainStep(t, n, samples_per_ray_capacity=128, error_map=em2)
    for _ in range(2):
        fs.step(o, d, gt, noise=noise, ray_w=w, img_idxs=img, pix_idxs=pix)
    torch.cuda.synchronize()
    assert int(em2.cnt.sum()) == 2 * n
    with pytest.raises(ValueError, match="ray_w"):
        fs.step(o, d, gt)
    bank = torch.rand(6, 64 * 64, 3, device=DEV)
    from datasets.synthetic import SyntheticLego
    ds = SyntheticLego(n_images=6, img_wh=(64, 64), focal=88.9, scene='random', with_rgb=False)
    fs.attach_ray_source(bank, ds.poses, ds.directions, seed=1)
    loss = fs.step_sampled()
    assert np.isfinite(float(loss)) and int(em2.cnt.sum()) == 3 * n
    plain = StaticTrainStep(NGPTrainer(_model(lego_bitfield), lr=1e-2), n, samples_per_ray_capacity=128)
    plain.attach_ray_source(bank, ds.poses, ds.directions, seed=1)
    _report("kernels per replay off / on (host-fed, sampled)",
            (plain.kernels_per_replay, fs.kernels_per_replay, plain.kernels_per_replay_sampled,
             fs.kernels_per_replay_sampled))
    assert fs.kernels_per_replay == plain.kernels_per_replay + 2
    assert fs.kernels_per_replay_sampled == plain.kernels_per_replay_sampled + 3
    with pytest.raises(ValueError, match="error map covers"):
        fs.attach_ray_source(bank[:5], ds.poses[:5], ds.directions, seed=1)


def test_skewed_map_graph_gradient_matches_module_path(lego_bitfield, monkeypatch):
    """Weights up to 1/alpha = 5: the graph step's gradient (weight kernel on the per-sample gradients) against the module
    path's (weighted MSE through autograd).  The two paths already differ without weights (fp16 autograd against the
    fused head, atomic order), so the bound is relative to that unweighted difference."""
    import torch
    from taichi_nerfs_b200.trainer import NGPTrainer
    n = 4096
    batch = _batch(n, 6)
    o, d, img, pix, gt, noise = batch
    em = _map((6, 64, 64, 16), _skewed_E(6 * 256, np.random.default_rng(4), hot=0.05))
    _, _, w = em.draw(n, 0)
    assert float(w.max()) > 2 and float(w.min()) < 0.5

    def module(ray_w):
        t = NGPTrainer(_model(lego_bitfield), lr=1e-2)
        monkeypatch.setattr(torch, 'rand_like', lambda x, **kw: noise.clone())
        t.forward_backward(o, d, gt, ray_w=ray_w)
        monkeypatch.undo()
        torch.cuda.synchronize()
        return t.flat_grad.clone()

    rel = {}
    for name, ww in (("uniform", torch.ones_like(w)), ("skewed", w)):
        g_graph = _graph_stages(lego_bitfield, batch, _map((6, 64, 64, 16)), ww)[3]
        g_mod = module(ww)
        rel[name] = float((g_graph - g_mod).norm() / g_mod.norm())
    _report("relative L2 difference graph vs module gradient (uniform weights, skewed weights)", rel)
    assert rel["skewed"] <= max(4 * rel["uniform"], 1e-3)


def test_every_model_kind_steps(lego_bitfield):
    """One graph step (host-fed) and one module step with error-map weights for the hash, tri-plane and voxel-grid
    models: both run and stay finite."""
    import torch
    from modules.networks import NGP
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    n = 2048
    o, d, img, pix, gt, noise = _batch(n, 9)
    em = _map((6, 64, 64, 16), _skewed_E(6 * 256, np.random.default_rng(1), hot=0.05))
    _, _, w = em.draw(n, 0)
    bits = torch.from_numpy(lego_bitfield)

    def make(kind):
        torch.manual_seed(0)
        if kind == "svox":
            m = VoxelGrid(scale=0.5, grid_size=97, grid_radius=0.0125, sh_degree=2).to(DEV)
            with torch.no_grad():
                m.density_fields.uniform_(-10, 50)
                m.sh_fields.uniform_(-1, 1)
        else:
            m = NGP(scale=0.5, max_res=1024, half_opt=kind == "hash", pos_encoder_type=kind).to(DEV)
        with torch.no_grad():
            m.density_bitfield.copy_(bits)
        return m

    for kind in ("hash", "triplane", "svox"):
        t = NGPTrainer(make(kind), lr=1e-2)
        fs = StaticTrainStep(t, n, samples_per_ray_capacity=256, error_map=em)
        loss = fs.step(o, d, gt, noise=noise, ray_w=w, img_idxs=img, pix_idxs=pix)
        p = torch.cat([q.detach().reshape(-1) for q in t.params])
        assert np.isfinite(float(loss)) and bool(torch.isfinite(p).all()), kind
        t2 = NGPTrainer(make(kind), lr=1e-2)
        loss2, res = t2.step(o, d, gt, ray_w=w)
        em.accumulate(res['rgb'].float(), gt, img, pix)
        p2 = torch.cat([q.detach().reshape(-1) for q in t2.params])
        assert np.isfinite(float(loss2.detach())) and bool(torch.isfinite(p2).all()), kind
    em.rebuild()
    assert bool(torch.isfinite(em.as_image()).all())


# ---- behaviour on the teacher Lego ---------------------------------------------------------------------------------
def test_teacher_lego_draws_the_object_and_keeps_psnr():
    """After 500 steps the map draws rays that see the object (target not pure white) at least twice as often as
    uniform sampling does; after 3000 steps the held-out PSNR is not below uniform sampling's minus MARGIN_DB."""
    from taichi_nerfs_b200.psnr import train_vs_teacher
    from datasets.teacher import load_teacher
    teacher = load_teacher(DEV)
    if teacher is None:
        pytest.skip("teacher model not staged")
    r500 = train_vs_teacher(DEV, steps=500, teacher=teacher, ray_sampling='error_map')
    em = r500["error_map"]
    from datasets.teacher import TeacherLego
    ds = TeacherLego(n_images=48, split='train', downsample=0.5, seed=23).to(DEV)
    ds_bank = ds.build_image_bank(teacher)
    obj = (ds_bank < 1.0).any(-1)               # [n_img, H*W]: the pixel sees the object
    img, pix, _ = em.draw(1 << 16, 500)
    share_map = float(obj[img, pix].float().mean())
    share_uniform = float(obj.float().mean())
    _report("share of object rays: error map / uniform", (share_map, share_uniform))
    assert share_map >= 2 * share_uniform
    a = train_vs_teacher(DEV, steps=3000, teacher=teacher)
    b = train_vs_teacher(DEV, steps=3000, teacher=teacher, ray_sampling='error_map')
    _report("held-out PSNR after 3000 steps: all_images / error_map", (a["psnr"], b["psnr"]))
    assert b["psnr"] >= a["psnr"] - MARGIN_DB


MARGIN_DB = 0.5
