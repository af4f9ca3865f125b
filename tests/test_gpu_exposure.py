"""Per-image exposure compensation (--exposure_lr, DESIGN.md §6k) on the GPU:

- ngp_exposure_apply against fp64 2^e c within one rounding of the row dtype (fp16 and fp32 rows, exposures in +-2
  stops, many images and one broadcast index), and bit for bit the input at e = 0;
- ngp_exposure_bwd against torch.autograd in fp64: the rewritten per-sample gradient within one rounding, the per-image
  gradient within k u sum|terms|; fp16 overflow and NaN raise found_inf;
- ngp_exposure_adam against the restatement (tests/exposure_ref.py) for several hyper states, the inf-skip, and the
  zero mean after the projection;
- the graph step's per-image gradient against the module path's for the fp16 hash model, the tri-plane model, the voxel
  grid and the device-sampled step;
- exposure on at learning rate 0 against exposure off: per-ray outputs and per-sample gradients bit for bit, and the
  kernel count;
- recovery of injected exposures on the teacher Lego, and train.py end to end.

Every bound prints the value measured beside it (pytest -s)."""
import json
import re

import numpy as np
import pytest

import exposure_ref as ref

pytestmark = pytest.mark.gpu

DEV = "cuda"
U32 = 2.0 ** -24
U_ROW = {"float32": 2.0 ** -24, "float16": 2.0 ** -11}
TINY = {"float32": 2.0 ** -150, "float16": 2.0 ** -25}   # half the spacing of the dtype's subnormals


def _report(name, value):
    print(f"measured {name}: {value}")


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def _T(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t if dtype is None else t.to(dtype)


def _rays_a(rng, n, max_cnt=40):
    """(ray, start, count) rows in shuffled order: some rays with 0 samples.  Returns rays_a, S and each row's ray."""
    counts = rng.integers(0, max_cnt, n)
    counts[rng.integers(0, n, n // 10)] = 0
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    order = rng.permutation(n)
    ra = np.stack([order, starts[order], counts[order]], 1).astype(np.int32)
    S = int(counts.sum())
    row_ray = np.repeat(np.arange(n), counts)   # rays are numbered by their start here
    return ra, S, row_ray


def _expo(rng, n_img, lo=-2.0, hi=2.0):
    e = np.zeros((n_img, 4), np.float32)
    e[:, :3] = rng.uniform(lo, hi, (n_img, 3))
    e[0, :3] = 0.0   # one image at exactly e = 0
    return e


# ---- apply ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("one_image", [False, True])
def test_apply_within_one_rounding_of_fp64(lib, dtype, one_image):
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(1)
    n, n_img = 5000, 1 if one_image else 37
    ra, S, _ = _rays_a(rng, n)
    e = _expo(rng, n_img)
    if one_image:
        e[0, :3] = [1.5, -0.75, -2.0]
    img = np.array([0]) if one_image else rng.integers(0, n_img, n)
    c = torch.rand(S, 3, device=DEV).to(getattr(torch, dtype))
    out = ops.exposure_apply(c, _T(ra), _T(img), _T(e))
    want = ref.apply(c.double().cpu().numpy(), ra, img, e)
    got = out.double().cpu().numpy()
    err = np.abs(got - want)
    _report(f"apply {dtype} one_image={one_image}: max |error| / (u |c'|)",
            float((err / (U_ROW[dtype] * np.abs(want)).clip(1e-300)).max()))
    # round to nearest of the exact product: at most half an ulp (u relative, or half a subnormal step)
    assert (err <= U_ROW[dtype] * np.abs(want) + TINY[dtype]).all()
    # e = 0: the input bit for bit
    z = ops.exposure_apply(c, _T(ra), _T(img), torch.zeros(n_img, 4, device=DEV))
    assert torch.equal(z.view(torch.int16 if dtype == "float16" else torch.int32),
                       c.view(torch.int16 if dtype == "float16" else torch.int32))


def test_apply_clamps_indices_and_reads_the_device_row_count(lib):
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(2)
    n, n_img = 3000, 5
    ra, S, _ = _rays_a(rng, n)
    e = _expo(rng, n_img)
    c = torch.rand(S, 3, device=DEV)
    img = rng.integers(-3, n_img + 3, n)
    got = ops.exposure_apply(c, _T(ra), _T(img), _T(e))
    want = ops.exposure_apply(c, _T(ra), _T(np.clip(img, 0, n_img - 1)), _T(e))
    assert torch.equal(got, want)
    # rows at or past the device count are not written
    cut = S - 123
    out = torch.full_like(c, -7.0)
    ops.exposure_apply(c, _T(ra), _T(img), _T(e), out=out,
                       n_rows_dev=torch.tensor([cut], device=DEV, dtype=torch.int32))
    torch.cuda.synchronize()
    assert bool((out[cut:] == -7.0).all())
    full = ref.apply(c.double().cpu().numpy(), ra, np.clip(img, 0, n_img - 1), e)
    wrote = ~np.isnan(ref.apply(c.double().cpu().numpy()[:cut], ra, np.clip(img, 0, n_img - 1), e))
    o = out[:cut].double().cpu().numpy()
    assert np.abs(o[wrote] - full[:cut][wrote]).max() <= U32 * np.abs(full[:cut][wrote]).max()


# ---- backward -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("one_image", [False, True])
def test_bwd_against_autograd(lib, dtype, one_image):
    """L = sum_s d_s . c'_s with c'_s = 2^e c_s in fp64 autograd: dL/dc and dL/de.

    The per-image sum is bounded by (u_row + k u) sum|terms| with k = ceil(n / 4) + ceil(max count / 32) + 12: the
    recursive-summation bound of the kernel's order (a lane's rows, five shuffle levels, the ln2 product, up to 4 rays
    in registers, then at most one atomic per 4 rays), plus the row dtype's rounding of c'."""
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(3)
    n, n_img = 5000, 1 if one_image else 23
    ra, S, _ = _rays_a(rng, n)
    e = _expo(rng, n_img)
    img = np.array([0]) if one_image else rng.integers(0, n_img, n)
    if one_image:
        e[0, :3] = [0.7, -1.3, 1.9]
    dt = getattr(torch, dtype)
    c = torch.rand(S, 3, device=DEV).to(dt)
    d = (torch.randn(S, 3, device=DEV) * 3).to(dt)
    out = ops.exposure_apply(c, _T(ra), _T(img), _T(e))
    dd = d.clone()
    grad = torch.zeros(n_img, 4, device=DEV)
    fi = torch.zeros(1, device=DEV, dtype=torch.int32)
    ops.exposure_bwd(out, dd, _T(ra), _T(img), _T(e), grad, found_inf=fi)
    assert int(fi) == 0
    # fp64 autograd
    row_id = np.empty(S, np.int64)   # each row's ray id
    for r, s0, k in ra.tolist():
        row_id[s0:s0 + k] = r
    row_img = torch.as_tensor(np.zeros(S, np.int64) if one_image else np.asarray(img)[row_id], device=DEV)
    et = torch.tensor(e[:, :3], device=DEV, dtype=torch.float64, requires_grad=True)
    ct = c.double().requires_grad_(True)
    cp = torch.exp2(et[row_img]) * ct
    (d.double() * cp).sum().backward()
    want_dc, want_ge = ct.grad, et.grad
    # the rewritten per-sample gradient: one rounding
    err_dc = (dd.double() - want_dc).abs() - TINY[dtype]
    err_dc = (err_dc / want_dc.abs().clamp_min(1e-300)).max()
    terms = (np.log(2.0) * d.double() * out.double()).abs()
    mag = torch.zeros(n_img, 3, device=DEV, dtype=torch.float64).index_add_(0, row_img, terms)
    k = -(-n // 4) + -(-int(ra[:, 2].max()) // 32) + 12
    bound = (U_ROW[dtype] + k * U32) * mag
    err_g = (grad[:, :3].double() - want_ge).abs()
    _report(f"bwd {dtype} one_image={one_image}: dL/dc max relative error / u_row, per-image |err| / (u sum|t|) max, "
            f"k", (float(err_dc / U_ROW[dtype]), float((err_g / (U32 * mag)).max()), k))
    assert float(err_dc) <= U_ROW[dtype]
    assert bool((err_g <= bound).all())
    assert bool((grad[:, 3] == 0).all())


@pytest.mark.parametrize("case", ["fp16_overflow", "nan"])
def test_bwd_raises_found_inf(lib, case):
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(4)
    n, n_img = 2000, 3
    ra, S, _ = _rays_a(rng, n)
    e = np.zeros((n_img, 4), np.float32)
    img = rng.integers(0, n_img, n)
    c = torch.rand(S, 3, device=DEV).half()
    d = torch.randn(S, 3, device=DEV).half()
    fi = torch.zeros(1, device=DEV, dtype=torch.int32)
    out = ops.exposure_apply(c, _T(ra), _T(img), _T(e))
    ops.exposure_bwd(out, d.clone(), _T(ra), _T(img), _T(e), torch.zeros(n_img, 4, device=DEV), found_inf=fi)
    assert int(fi) == 0
    if case == "fp16_overflow":
        e[:, :3] = 1.0                      # g = 2: 60000 -> 120000 overflows fp16
        d[int(ra[ra[:, 2] > 0][0, 1])] = 60000.0
    else:
        d[int(ra[ra[:, 2] > 0][0, 1]), 1] = float("nan")
    out = ops.exposure_apply(c, _T(ra), _T(img), _T(e))
    dd = d.clone()
    ops.exposure_bwd(out, dd, _T(ra), _T(img), _T(e), torch.zeros(n_img, 4, device=DEV), found_inf=fi)
    assert int(fi) == 1
    assert not bool(torch.isfinite(dd.float()).all())


# ---- Adam -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_img", [1, 7, 1000])
def test_adam_against_the_restatement(lib, n_img):
    """Several hyper states (first step, a late step, a small loss scale), applied in sequence.  Each exposure is
    within 16 u (|e'| + |step|) of the fp64 restatement plus the same bound averaged over the images (the mean the
    projection subtracts); the moments within 8 u; the per-channel mean within N u max|e| of zero."""
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(5)
    b1, b2, eps = 0.9, 0.99, 1e-15
    states = [(1e-2 / (1 - b1), np.sqrt(1 - b2), 2.0 ** -16, 0.1),
              (3e-3 / (1 - b1 ** 500), np.sqrt(1 - b2 ** 500), 2.0 ** -19, 1.0),
              (1e-2, 1.0, 1.0, 0.03)]
    e = _expo(rng, n_img, -0.5, 0.5)
    e[:, :3] -= e[:, :3].mean(0)
    m = np.zeros((n_img, 4), np.float32)
    v = np.zeros((n_img, 4), np.float32)
    m[:, :3] = rng.standard_normal((n_img, 3)) * 1e-2
    v[:, :3] = rng.random((n_img, 3)) * 1e-4
    worst = 0.0
    for lr_bc1, bc2, inv, ratio in states:
        g = np.zeros((n_img, 4), np.float32)
        g[:, :3] = rng.standard_normal((n_img, 3)) / inv * 1e-2
        E, G, M, V = (_T(x.copy()) for x in (e, g, m, v))
        hyper = torch.tensor([lr_bc1, bc2, inv, 0.0], device=DEV, dtype=torch.float32)
        ops.exposure_adam(E, G, M, V, hyper, ratio, beta1=b1, beta2=b2, eps=eps)
        hy = hyper.double().cpu().numpy()   # the fp32 scalars the kernel reads
        args = (e[:, :3], g[:, :3], m[:, :3], v[:, :3], hy, float(np.float32(ratio)), b1, b2, eps)
        we, _, wm, wv = ref.adam(*args)
        pre = ref.adam(*args, project=False)[0]
        scale = np.abs(pre) + np.abs(pre - e[:, :3])
        bound = 16 * U32 * (scale + scale.mean(0))
        ge = E.cpu().numpy().astype(np.float64)
        err = np.abs(ge[:, :3] - we)
        worst = max(worst, float((err / bound).max()))
        assert (err <= bound).all()
        assert np.abs(M.cpu().numpy()[:, :3] - wm).max() <= 8 * U32 * np.abs(wm).max()
        assert np.abs(V.cpu().numpy()[:, :3] - wv).max() <= 8 * U32 * np.abs(wv).max()
        assert not G.any() and not E[:, 3].any()
        mean = np.abs(ge[:, :3].mean(0))
        assert (mean <= n_img * U32 * np.abs(ge[:, :3]).max(0)).all(), mean
        e, m, v = E.cpu().numpy(), M.cpu().numpy(), V.cpu().numpy()
    _report(f"adam n_img={n_img}: max |err| / bound", worst)


def test_adam_skips_on_found_inf_and_keeps_zero_exposures_at_rate_zero(lib):
    import torch
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(6)
    n_img = 300
    e = _expo(rng, n_img, -0.3, 0.3)
    E, G, M, V = _T(e.copy()), _T(np.full((n_img, 4), np.inf, np.float32)), _T(e * 0.1), _T(np.abs(e) * 0.01)
    hyper = torch.tensor([0.1, 0.3, 1.0, 0.0], device=DEV)
    fi = torch.ones(1, device=DEV, dtype=torch.int32)
    m0, v0 = M.clone(), V.clone()
    ops.exposure_adam(E, G, M, V, hyper, 1.0, found_inf=fi)
    assert torch.equal(E, _T(e)) and torch.equal(M, m0) and torch.equal(V, v0) and not G.any()
    # rate 0 at e = 0: exactly 0 after the update and the projection
    Z = torch.zeros(n_img, 4, device=DEV)
    G = torch.randn(n_img, 4, device=DEV)
    ops.exposure_adam(Z, G, torch.zeros_like(Z), torch.zeros_like(Z), hyper, 0.0)
    assert not Z.any() and not G.any()


# ---- the training step ----------------------------------------------------------------------------------------------
def _batch(n, seed, n_img=6, wh=64):
    import torch
    from datasets.ray_utils import get_rays
    from datasets.synthetic import SyntheticLego
    ds = SyntheticLego(n_images=n_img, img_wh=(wh, wh), focal=88.9, scene='random', with_rgb=False)
    g = torch.Generator().manual_seed(seed)
    pix = torch.randint(0, wh * wh, (n,), generator=g)
    img = torch.randint(0, n_img, (n,), generator=g)
    o, d = get_rays(ds.directions[pix], ds.poses[img])
    return (o.to(DEV).contiguous(), d.to(DEV).contiguous(), img.to(DEV), torch.rand(n, 3, generator=g).to(DEV),
            torch.rand(n, generator=g).to(DEV)), ds


def _model(kind, lego_bitfield):
    import torch
    from modules.networks import NGP
    from modules.voxel_grid import VoxelGrid
    torch.manual_seed(3)
    if kind == "svox":
        m = VoxelGrid(scale=0.5, grid_size=97, grid_radius=0.0125, sh_degree=2).to(DEV)
        with torch.no_grad():
            m.density_fields.uniform_(-10, 50)
            m.sh_fields.uniform_(-1, 1)
    else:
        m = NGP(scale=0.5, max_res=1024, half_opt=kind == "hash", pos_encoder_type=kind).to(DEV)
        if kind == "hash":
            with torch.no_grad():
                m.pos_encoder.hash_table.mul_(2e3)
    with torch.no_grad():
        m.density_bitfield.copy_(torch.from_numpy(lego_bitfield))
    return m


def _exposure(n_img, seed, ratio=0.1):
    from taichi_nerfs_b200.exposure import ExposureCorrection
    x = ExposureCorrection(n_img, ratio, DEV)
    e = _expo(np.random.default_rng(seed), n_img, -0.5, 0.5)
    e[:, :3] -= e[:, :3].mean(0)
    x.exposure.copy_(_T(e))
    return x


def _graph_grad(kind, lego_bitfield, batch, expo, sampled_src=None):
    """The graph step's stages enqueued eagerly (no update): the exposure gradient and the step."""
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    o, d, img, gt, noise = batch
    n = o.shape[0]
    t = NGPTrainer(_model(kind, lego_bitfield), lr=1e-2, exposure=expo)
    fs = StaticTrainStep(t, n, samples_per_ray_capacity=256, use_graph=False)
    if sampled_src is not None:
        fs.attach_ray_source(*sampled_src, seed=5)
        fs._enqueue_sampler()
    else:
        for k, v in (("rays_o", o), ("rays_d", d), ("gt", gt), ("noise", noise)):
            getattr(fs, k).copy_(v)
        fs.expo_img.copy_(img)
    fs.counter.zero_()
    fs.loss_sum.zero_()
    t.found_inf.zero_()
    fs._enqueue_march()
    fs._enqueue_network()
    torch.cuda.synchronize()
    assert int(fs.counter[1]) == 0 and int(t.found_inf) == 0
    return expo.grad[:, :3].double().cpu().numpy().copy(), fs


def _module_grad(kind, lego_bitfield, batch, expo, monkeypatch):
    import torch
    from taichi_nerfs_b200.trainer import NGPTrainer
    o, d, img, gt, noise = batch
    t = NGPTrainer(_model(kind, lego_bitfield), lr=1e-2, exposure=expo)
    monkeypatch.setattr(torch, 'rand_like', lambda x, **kw: noise.clone())
    t.forward_backward(o, d, gt, img_idxs=img)
    monkeypatch.undo()
    torch.cuda.synchronize()
    return expo.grad[:, :3].double().cpu().numpy().copy()


GRAPH_VS_MODULE = 1e-4   # max |g_graph - g_module| over max |g_module|, per channel (measured <= 2.5e-7)


@pytest.mark.parametrize("kind", ["hash", "triplane", "svox", "sampled"])
def test_graph_step_exposure_gradient_matches_the_module_path(lego_bitfield, monkeypatch, kind):
    """One seeded batch through both paths.  They already differ without exposure (fp16 autograd against the fused
    head, the two marches' row order), so the bound is a relative one: GRAPH_VS_MODULE of the largest per-image
    gradient of each channel."""
    import torch
    from taichi_nerfs_b200 import ops
    n = 4096
    batch, ds = _batch(n, 7)
    src = None
    model_kind = "hash" if kind == "sampled" else kind
    if kind == "sampled":   # the batch the device sampler draws at step 0 (noise included)
        bank = torch.rand(6, 64 * 64, 3, device=DEV)
        src = (bank, ds.poses.to(DEV), ds.directions.to(DEV))
        r = ops.sample_ray_batch(bank, src[1], src[2], n, seed=5, step=0, return_indices=True)
        batch = (r["rays_o"], r["rays_d"], r["img_idxs"], r["rgb"], r["noise"])
    g_graph, fs = _graph_grad(model_kind, lego_bitfield, batch, _exposure(6, 8), src)
    if kind == "sampled":
        assert torch.equal(fs.expo_img, batch[2]) and torch.equal(fs.rays_d, batch[1])
    g_mod = _module_grad(model_kind, lego_bitfield, batch, _exposure(6, 8), monkeypatch)
    scale = np.abs(g_mod).max(0)
    rel = np.abs(g_graph - g_mod).max(0) / scale
    _report(f"{kind}: graph vs module exposure gradient, max |diff| / max |g| per channel", rel.tolist())
    assert (scale > 0).all() and rel.max() <= GRAPH_VS_MODULE


def _stages(lego_bitfield, batch, expo):
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    o, d, img, gt, noise = batch
    n = o.shape[0]
    t = NGPTrainer(_model("hash", lego_bitfield), lr=1e-2, exposure=expo)
    fs = StaticTrainStep(t, n, samples_per_ray_capacity=128, use_graph=False)
    for k, v in (("rays_o", o), ("rays_d", d), ("gt", gt), ("noise", noise)):
        getattr(fs, k).copy_(v)
    if expo is not None:
        fs.expo_img.copy_(img)
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
    for k in ("xyzs", "ts", "deltas", "sig", "rgbs", "dsig", "drgbs", "demb"):
        out[k] = getattr(fs, k)[rows].clone()
    if expo is not None:
        assert torch.equal(fs.rgbs_expo[rows], out["rgbs"])   # e = 0: the head read the network's colours
    return out, int(t.found_inf), S


def test_flag_off_is_unchanged(lego_bitfield):
    """Exposure on at learning rate 0 against off on the same rays: every per-ray output and every per-sample buffer
    (the colours, their rewritten gradients, dL/demb) gathered in ray order bit for bit; three graph replays keep the
    exposures at exactly 0 with no step skipped; the graph gains exactly the three exposure nodes (apply, backward,
    Adam) on the hash model, whose backward raises found_inf itself."""
    import torch
    from taichi_nerfs_b200.exposure import ExposureCorrection
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    n = 4096
    batch, _ = _batch(n, 9)
    on, f_on, S = _stages(lego_bitfield, batch, ExposureCorrection(6, 0.0, DEV))
    off, f_off, S_off = _stages(lego_bitfield, batch, None)
    assert S == S_off and S > 20000 and f_on == f_off == 0
    for k in on:
        assert torch.equal(on[k], off[k]), k
    o, d, img, gt, noise = batch
    x = ExposureCorrection(6, 0.0, DEV)
    t = NGPTrainer(_model("hash", lego_bitfield), lr=1e-2, exposure=x)
    fs = StaticTrainStep(t, n, samples_per_ray_capacity=128)
    for _ in range(3):
        fs.step(o, d, gt, noise=noise, img_idxs=img)
    torch.cuda.synchronize()
    assert not x.exposure.any() and not x.grad.any()
    assert int(t.hyper[3:4].view(torch.int32)) == 3   # Adam's applied-step count: no step skipped
    plain = StaticTrainStep(NGPTrainer(_model("hash", lego_bitfield), lr=1e-2), n, samples_per_ray_capacity=128)
    _report("kernels per replay off / on", (plain.kernels_per_replay, fs.kernels_per_replay))
    assert fs.kernels_per_replay == plain.kernels_per_replay + 3
    # argument checks: img_idxs is required with exposure, and still refused without any per-image feature
    with pytest.raises(ValueError, match="img_idxs"):
        fs.step(o, d, gt)
    with pytest.raises(ValueError, match="img_idxs"):
        plain.step(o, d, gt, img_idxs=img)
    with pytest.raises(ValueError, match="img_idxs"):
        t.step(o, d, gt)


# ---- recovery on the teacher Lego -----------------------------------------------------------------------------------
# 24 training views of the teacher at 200 x 200; each image's foreground scaled by a seeded per-channel exposure,
# uniform in +-0.5 stops with zero mean per channel: gt = 2^e (rgb - (1 - op)) + (1 - op).  Test views are clean.
# --half_opt graph step, 8192 rays, RECOVERY_STEPS steps, --exposure_lr 1e-3 (lr 1e-2) against exposure off.
RECOVERY_STEPS = 3000
STOPS = 0.5


def _train_teacher(ds, with_exposure, steps):
    import torch
    from modules.networks import NGP
    from modules.rendering import MAX_SAMPLES
    from datasets.ray_utils import get_rays
    from taichi_nerfs_b200.exposure import ExposureCorrection
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    torch.manual_seed(23)
    model = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    x = ExposureCorrection(len(ds.poses), 1e-3 / 1e-2, DEV) if with_exposure else None
    tr = NGPTrainer(model, lr=1e-2, max_steps=steps, exposure=x)
    fs = StaticTrainStep(tr, ds.batch_size)
    for step in range(steps + 1):
        data = ds[step]
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            if step % 16 == 0:
                model.update_density_grid(0.01 * MAX_SAMPLES / 3 ** 0.5, warmup=step < 256)
        o, d = get_rays(data['direction'], data['pose'])
        fs.step(o, d, data['rgb'], img_idxs=data['img_idxs'] if with_exposure else None)
    return model, x


def _held_out_psnr(model, test):
    import torch
    import torch.nn.functional as F
    from datasets.ray_utils import get_rays
    from modules.rendering import render
    ps = []
    with torch.no_grad():
        for i in range(len(test)):
            td = test[i]
            with torch.autocast(device_type='cuda', dtype=torch.float16):
                o, d = get_rays(test.directions, td['pose'])
                res = render(model, o, d, test_time=True)
            ps.append(float(-10 * torch.log10(F.mse_loss(res['rgb'].float(), td['rgb']))))
    return float(np.mean(ps))


def test_recovery_on_the_teacher_lego():
    import torch
    from datasets.ray_utils import get_rays
    from datasets.teacher import TeacherLego, load_teacher, teacher_dir
    from modules.rendering import render
    if teacher_dir() is None:
        pytest.skip("teacher model not staged (__graft_entry__.build())")
    ds = TeacherLego(n_images=24, img_wh=(200, 200), focal=277.78, batch_size=8192).to(DEV)
    ds.build_image_bank()
    test = TeacherLego(n_images=4, img_wh=(200, 200), focal=277.78, split='test').to(DEV)
    test.build_image_bank()
    teacher = load_teacher(DEV)
    rng = np.random.default_rng(2026)
    inj = rng.uniform(-STOPS, STOPS, (24, 3))
    inj -= inj.mean(0)
    with torch.no_grad():
        for i in range(24):
            o, d = get_rays(ds.directions, ds.poses[i])
            with torch.autocast('cuda', dtype=torch.float16):
                op = render(teacher, o, d, test_time=True, T_threshold=1e-2, exp_step_factor=0.0)['opacity']
            bg = (1 - op.float().clamp(0, 1))[:, None]
            g = torch.tensor(np.exp2(inj[i]), device=DEV, dtype=torch.float32)
            ds.images[i] = g * (ds.images[i] - bg) + bg
    res = {"injected rms (stops)": float(np.sqrt((inj ** 2).mean()))}
    m_off, _ = _train_teacher(ds, False, RECOVERY_STEPS)
    res["psnr without exposure"] = _held_out_psnr(m_off, test)
    del m_off
    m_on, x = _train_teacher(ds, True, RECOVERY_STEPS)
    res["psnr with exposure"] = _held_out_psnr(m_on, test)
    got = x.exposures().astype(np.float64)
    res["recovered rms error (stops)"] = float(np.sqrt(((got - inj) ** 2).mean()))
    res["recovered per-channel mean"] = got.mean(0).tolist()
    _report("teacher Lego exposure recovery", json.dumps(res))
    assert res["psnr with exposure"] > res["psnr without exposure"], res
    assert res["recovered rms error (stops)"] <= 0.5 * res["injected rms (stops)"], res


# ---- train.py end to end --------------------------------------------------------------------------------------------
def test_train_py_with_exposure(tmp_path, monkeypatch, capsys):
    import train
    from datasets.teacher import teacher_dir
    if teacher_dir() is None:
        pytest.skip("teacher model not staged (__graft_entry__.build())")
    monkeypatch.chdir(tmp_path)
    psnrs = train.main(['--dataset_name', 'teacher', '--downsample', '0.125', '--half_opt', '--graph_step',
                        '--max_steps', '400', '--exposure_lr', '1e-3'])
    out = capsys.readouterr().out
    line = [ln for ln in out.splitlines() if ln.startswith("exposure:")][-1]
    mean_abs, max_abs = (float(v) for v in re.findall(r"= ([0-9.e+-]+) stops", line)[:2])
    E = np.load(tmp_path / 'results' / 'exposures.npy')
    with capsys.disabled():
        _report("train.py exposure: psnr, mean |e|, max |e|, per-channel mean", (psnrs, mean_abs, max_abs,
                                                                                  E.mean(0).tolist()))
    assert E.dtype == np.float32 and E.shape == (48, 3) and np.isfinite(E).all()
    assert (np.abs(E.astype(np.float64).mean(0)) < 1e-5).all()
    assert 0 <= mean_abs <= max_abs
    assert min(psnrs) > 15.0
