"""The tri-plane encoder on the GPU against the CPU oracle: kernels (bit-exact forward, backward), the model's fused
MLP path, one training step, the occupancy-grid update, whole frames, train.py end to end and PSNR on the teacher."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import train_step as TS
from oracle import triplane as OT
from taichi_nerfs_b200.layout import make_triplane_layout

pytestmark = pytest.mark.gpu

DEV = "cuda"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def _positions(rng, n, lay):
    """Random points, points on cell boundaries of every level, 0 and 1, and points slightly outside [0, 1]."""
    pts = [rng.random((n, 3), dtype=np.float32)]
    for level in range(lay.levels):
        r = lay.resolutions[level]
        k = rng.integers(0, r, (64, 3)).astype(np.float32)
        pts.append(((k + np.float32(0.5)) / np.float32(r - 1)).clip(0, 1).astype(np.float32))
    pts.append(np.array([[0, 0, 0], [1, 1, 1], [0, 1, 0.5], [1, 0, 1]], np.float32))
    out = (rng.random((256, 3), dtype=np.float32) * np.float32(1.004) - np.float32(0.002)).astype(np.float32)
    pts.append(out)
    return np.concatenate(pts)


@pytest.mark.parametrize("levels,F,max_res", [(8, 4, 1024), (8, 4, 4096), (16, 2, 2048)])
def test_forward_bit_exact_vs_oracle(levels, F, max_res):
    from taichi_nerfs_b200 import _lib, ops
    rng = np.random.default_rng(max_res + F)
    lay = make_triplane_layout(levels, 16, max_res, F)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    xyz = _positions(rng, 20000, lay)
    ref = OT.triplane_encode_fwd(xyz, table, lay)
    tab = T(table)
    cl = lay.as_ctypes()
    out = ops.triplane_encode_fwd(T(xyz), tab, cl)
    assert np.array_equal(N(out).view(np.uint32), ref.view(np.uint32))
    # folded AABB normalisation == torch normalisation first (NGP.density, networks.py:144)
    lo = torch.full((1, 3), -0.5, device=DEV)
    hi = torch.full((1, 3), 0.5, device=DEV)
    xw = (T(rng.random((50000, 3), dtype=np.float32)) - 0.5) * 0.999
    a = ops.triplane_encode_fwd(xw, tab, cl, aabb=lo.flatten().tolist() + (hi - lo).flatten().tolist())
    b = ops.triplane_encode_fwd(((xw - lo) / (hi - lo)).contiguous(), tab, cl)
    assert torch.equal(a, b)
    # _dyn: the row count read on the device; rows >= it untouched
    n, k = xyz.shape[0], xyz.shape[0] // 3
    dyn = torch.full((n, lay.out_dim), -7.0, device=DEV)
    n_dev = torch.tensor([k], device=DEV, dtype=torch.int32)
    _lib.check(_lib.load().ngp_triplane_encode_fwd_dyn(ops._ptr(T(xyz)), ops._ptr(tab), ops.C.byref(cl), ops._ptr(dyn),
                                                        n, ops._ptr(n_dev), None, ops._stream()))
    assert torch.equal(dyn[:k], out[:k]) and bool((dyn[k:] == -7.0).all())


def _march_samples(n_rays, seed):
    """Sample positions of a real training march (Lego occupancy bitfield) in [0, 1]."""
    bits = np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"]
    o, d = TS.make_rays(n_rays, seed=seed)
    hits = O.ray_aabb_intersect(o, d, 0.5)
    noise = np.random.default_rng(seed).random(n_rays, dtype=np.float32)
    _, xyzs, _, _, _, S = O.raymarching_train(o, d, hits, bits, noise, 1, 0.5, 0.0, 128, 1024)
    lo, hi = np.float32(-0.5), np.float32(0.5)
    return ((xyzs[:S] - lo) / (hi - lo)).astype(np.float32)


def test_backward_vs_oracle_on_a_real_march():
    """>= 1 M samples of a real march; returned-gradient path and grad_sink path, within 1e-3 of max |G|."""
    from modules.triplane import TriPlaneEncoder
    xn = _march_samples(50000, seed=3)
    assert xn.shape[0] >= 1_000_000, xn.shape
    torch.manual_seed(0)
    enc = TriPlaneEncoder(base_res=16, max_res=1024, levels=8, feature_per_level=4).to(DEV)
    rng = np.random.default_rng(4)
    dout = rng.standard_normal((xn.shape[0], 32)).astype(np.float32)
    dout[rng.random(xn.shape[0]) < 0.2] = 0.0              # samples behind the termination point
    g_ref = OT.triplane_encode_bwd(xn, N(enc.plane_embedding), dout, enc._layout)
    scale = np.abs(g_ref).max()
    x = T(xn)
    emb = enc(x)
    assert np.array_equal(N(emb).view(np.uint32), OT.triplane_encode_fwd(xn, N(enc.plane_embedding), enc._layout)
                          .view(np.uint32))
    emb.backward(T(dout))
    g = N(enc.plane_embedding.grad)
    err = np.abs(g - g_ref).max()
    print("returned gradient: max err", err / scale, "rel")
    assert scale > 0 and err <= 1e-3 * scale
    sink = torch.zeros(enc.total_param_size, device=DEV)
    enc.plane_embedding.grad = None
    enc.grad_sink = sink
    enc(x).backward(T(dout))
    assert enc.plane_embedding.grad is None
    err = np.abs(N(sink) - g_ref).max()
    assert err <= 1e-3 * scale


def _triplane_model(seed=0, amp=1.6):
    from modules.networks import NGP
    torch.manual_seed(seed)
    m = NGP(scale=0.5, pos_encoder_type='triplane', max_res=1024).to(DEV)
    with torch.no_grad():
        m.pos_encoder.plane_embedding.mul_(2.0).sub_(1.0).mul_(amp)   # features of both signs, products up to amp^3
    return m


def test_fused_mlp_path_equals_torch_path_triplane():
    """NGP.forward of a tri-plane model through the fused MLP (fp32 embedding) vs the nn.Linear graph under autocast,
    with the tolerances of the hash model's test."""
    m = _triplane_model()
    x = (torch.rand(5000, 3, device=DEV) - 0.5) * 0.98
    d = torch.randn(5000, 3, device=DEV)
    with torch.autocast('cuda', dtype=torch.float16):
        s_f, c_f = m(x, d)
        m._fusable = lambda _x: False
        s_t, c_t = m(x, d)
    assert (s_f - s_t).abs().max() <= 8e-3 * s_t.abs().max()
    assert (c_f.float() - c_t.float()).abs().max() <= 3e-3


def _mlp_weights_np(m):
    from taichi_nerfs_b200.fused_mlp import mlp_weights
    return [N(w).copy() for w in mlp_weights(m)]


def test_training_step_matches_oracle():
    """One NGPTrainer step (render -> MSE -> backward -> fused Adam) against the oracle's full step."""
    from taichi_nerfs_b200.trainer import NGPTrainer
    m = _triplane_model(seed=1)
    bits = np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"]
    with torch.no_grad():
        m.density_bitfield.copy_(T(bits))
    table0, ws0 = N(m.pos_encoder.plane_embedding).copy(), _mlp_weights_np(m)
    n = 4096
    o, d = TS.make_rays(n, seed=3)
    gt = np.random.default_rng(3).random((n, 3), dtype=np.float32)
    real_rand_like = torch.rand_like
    torch.rand_like = lambda t, **k: torch.zeros_like(t)
    try:
        tr = NGPTrainer(m, lr=1e-2)
        assert m.pos_encoder.grad_sink is not None and tr._shadow_full is None
        loss, res = tr.forward_backward(T(o), T(d), T(gt))
    finally:
        torch.rand_like = real_rand_like
    P = m.pos_encoder.total_param_size
    g_table = N(tr.flat_grad[:P]).copy()
    g_mlp = np.concatenate([N(tr.flat_grad[off:off + s]) for off, s in tr.slices[1:]])
    tr.optimizer_step()
    torch.cuda.synchronize()

    om = OT.TriplaneOracleModel(m.pos_encoder._layout, table0, ws0, bits)
    rgb_ref, cache = OT.forward(om, o, d, np.zeros(n, np.float32))
    loss_ref, g_ref, g_mlp_ref = OT.backward(om, cache, rgb_ref, gt, tr.loss_scale)
    assert int(res["rm_samples"]) == cache["S"]
    assert abs(float(loss) - loss_ref) <= 1e-3 * loss_ref
    for g, r in ((g_table, g_ref), (g_mlp, g_mlp_ref)):
        s = np.abs(r).max()
        print("gradient max err", np.abs(g - r).max() / s, "rel")
        assert s > 0 and np.abs(g - r).max() <= 1e-3 * s
    TS.adam(om, g_ref, g_mlp_ref, 1e-2, tr.loss_scale)
    # Adam's first step moves every entry with a clear gradient by lr * sign(g); tiny gradients may differ in sign
    p_gpu = N(m.pos_encoder.plane_embedding)
    clear = np.abs(g_ref) > 1e-3 * np.abs(g_ref).max()
    assert clear.sum() > 1000
    assert np.abs(p_gpu - om.table)[clear].max() <= 1e-5
    assert np.abs(p_gpu - om.table).max() <= 2e-2 + 1e-5
    w_gpu = np.concatenate([w.reshape(-1) for w in _mlp_weights_np(m)])
    w_ref = np.concatenate([w.reshape(-1) for w in om.ws])
    clear = np.abs(g_mlp_ref) > 1e-3 * np.abs(g_mlp_ref).max()
    assert np.abs(w_gpu - w_ref)[clear].max() <= 1e-5


def test_update_density_grid_is_sync_free_and_matches_reference_statistics():
    """No host synchronisation in any update; the statistics of the warm-up updates (every cell evaluated once at a
    jittered position) equal those of the reference's op sequence.  The sampled updates are compared on the hash model
    only: they pick occupied cells with replacement, and duplicate picks keep the maximum here but an arbitrary one in
    the reference (DESIGN.md §2) - on the random tri-plane field, which varies strongly inside a cell, that moves the
    occupancy by a few percent (0.215 against 0.257 measured after a warm-up, 3 sampled and another warm-up
    update)."""
    thr = 0.01 * 1024 / 3 ** 0.5

    def fresh():
        return _triplane_model(seed=11, amp=3.0)
    a, b = fresh(), fresh()
    a.update_density_grid(thr, warmup=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.update_density_grid(thr, warmup=True)
        for _ in range(3):
            a.update_density_grid(thr, warmup=False)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    a = fresh()
    for _ in range(2):
        a.update_density_grid(thr, warmup=True)
        b.update_density_grid_reference(thr, warmup=True)
    occ_a = float(np.unpackbits(N(a.density_bitfield)).mean())
    occ_b = float(np.unpackbits(N(b.density_bitfield)).mean())
    print("occupancy", occ_a, occ_b)
    assert 0.02 < occ_a < 0.98 and abs(occ_a - occ_b) < 0.02, (occ_a, occ_b)
    ga, gb = N(a.density_grid.float()), N(b.density_grid.float())
    assert abs(ga.mean() - gb.mean()) < 0.02 * abs(gb.mean())


def _frame_case():
    from test_gpu_frame import _weights
    from taichi_nerfs_b200.fused_mlp import mlp_weights
    m = _triplane_model(seed=12, amp=3.0)
    rng = np.random.default_rng(13)
    ws = _weights(rng)
    bits = np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"].copy()
    with torch.no_grad():
        for p, w in zip(mlp_weights(m), ws):
            p.copy_(T(w))
        m.density_bitfield.copy_(T(bits))
    om = OT.TriplaneOracleModel(m.pos_encoder._layout, N(m.pos_encoder.plane_embedding), ws, bits)
    o, d = TS.make_rays(20000, seed=12)
    return m, om, o, d


@pytest.mark.parametrize("thr", [1e-4, 0.25])
def test_frames_match_oracle(thr):
    """FrameRenderer (render(test_time=True)) and render_frame against oracle render_test; graph replay == eager."""
    import modules.rendering as R
    from test_gpu_frame import _check_frame
    from taichi_nerfs_b200.render_frame import FrameRenderer, render_frame
    m, om, o, d = _frame_case()
    ref = OT.render_test(om, o, d, 0.0, thr)
    hits = O.ray_aabb_intersect(o, d, 0.5)
    with torch.autocast("cuda", dtype=torch.float16):
        out = R.render(m, T(o), T(d), test_time=True, exp_step_factor=0.0, T_threshold=thr)
    _check_frame(out, ref, hits, thr, f"triplane FrameRenderer thr={thr}")
    assert (ref["n_term"] < ref["rays_a"][:, 2]).mean() > 0.02        # early termination is exercised
    fr = m._frame_renderers[(o.shape[0], 0.0, float(thr), T(o).device)]
    assert fr.emb.dtype == torch.float32
    with torch.autocast("cuda", dtype=torch.float16):
        again = R.render(m, T(o), T(d), test_time=True, exp_step_factor=0.0, T_threshold=thr)
    eager = FrameRenderer(m, o.shape[0], 0.0, thr, use_graph=False).render(T(o), T(d))
    for k in ("opacity", "depth", "rgb", "total_samples"):
        assert torch.equal(out[k], again[k]) and torch.equal(out[k], eager[k]), k
    # render_frame: two-pass march on the first frame, single-pass march on the second
    for _ in range(2):
        with torch.autocast("cuda", dtype=torch.float16):
            rf = render_frame(m, T(o), T(d), 0.0, thr)
        _check_frame(rf, ref, hits, thr, f"triplane render_frame thr={thr}")
        assert int(rf["total_samples"]) == ref["S"]


def test_no_hash_kernel_is_reached(monkeypatch):
    """A tri-plane model never launches a hash-encoder kernel: forward/backward, grid update, both frame renderers."""
    from taichi_nerfs_b200 import _lib
    from taichi_nerfs_b200.render_frame import FrameRenderer, render_frame
    from taichi_nerfs_b200.trainer import NGPTrainer
    lib = _lib.load()
    for name in [s for s in _lib.EXPORTS if s.startswith("ngp_hash_encode")]:
        def boom(*a, _n=name, **k):
            raise AssertionError(f"{_n} called for a tri-plane model")
        monkeypatch.setattr(lib, name, boom)
    m, _, o, d = _frame_case()
    tr = NGPTrainer(m, lr=1e-2)
    tr.step(T(o[:2048]), T(d[:2048]), torch.rand(2048, 3, device=DEV))
    with torch.autocast("cuda", dtype=torch.float16):
        m.update_density_grid(0.01 * 1024 / 3 ** 0.5, warmup=True)
    FrameRenderer(m, 1000, use_graph=False).render(T(o[:1000]), T(d[:1000]))
    render_frame(m, T(o[:1000]), T(d[:1000]))


def test_train_main_end_to_end(tmp_path, monkeypatch):
    """train.main with --encoder_type triplane writes results/model.pth, which reloads through --ckpt_path;
    --graph_step with the tri-plane encoder is refused."""
    import train
    from test_gpu_e2e import _small_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _small_dataset})
    args = ['--dataset_name', 'synthetic', '--encoder_type', 'triplane', '--batch_size', '4096']
    psnrs = train.main(args + ['--max_steps', '300'])
    ckpt = tmp_path / 'results' / 'model.pth'
    assert ckpt.exists()
    sd = torch.load(ckpt, map_location='cpu')
    assert sd['pos_encoder.plane_embedding'].shape == (12_582_912,)
    print("triplane train.py psnr", psnrs)
    assert min(psnrs) > 25.0, psnrs          # measured 30.9 dB (H100 80GB HBM3, 700 W power limit)
    from modules.networks import NGP
    m = NGP(**train.build_model_config(train.get_opts(args)))
    m.load_state_dict(sd)
    assert torch.equal(m.pos_encoder.plane_embedding.detach(), sd['pos_encoder.plane_embedding'])
    # --ckpt_path resumes from it (one more step: Adam's first step moves every parameter by ~lr, so the PSNR drops)
    again = train.main(args + ['--max_steps', '1', '--ckpt_path', str(ckpt)])
    assert min(again) > 15.0, again
    with pytest.raises(SystemExit):
        train.main(args + ['--graph_step', '--max_steps', '1'])


def test_psnr_vs_teacher_triplane():
    """PSNR against the teacher after 1500 module-path steps (an untrained model scores about 9 dB).
    Measured once: 26.7 dB (views 25.4, 27.9) on an H100 80GB HBM3 at a 700 W power limit; the gate is 2 dB below."""
    from taichi_nerfs_b200.psnr import train_vs_teacher
    r = train_vs_teacher(torch.device('cuda'), steps=1500, train_views=32, test_views=2, downsample=0.25,
                         pos_encoder_type='triplane', graph=False)
    assert r is not None
    print("triplane psnr vs teacher", r["psnr"], r["psnr_views"])
    assert r["psnr"] >= 24.7, r["psnr_views"]
