"""SSIM on the GPU (`ngp_ssim` through `ops.ssim`, DESIGN.md §6e) against the fp64 restatement tests/ssim_ref.py
within its written per-image bound; determinism, CUDA-graph replay and non-finite inputs; a batch past 2^31 floats;
and the two callers, train.py's evaluation line and psnr.train_vs_teacher.

Each shape runs four images with different content: uniform noise with a correlated target, a smooth field,
near-constant patches (the variances sit far below C2, so C2 dominates the denominator) and predictions in
[-0.2, 1.3] (unclamped, as the evaluation passes them)."""
import re

import numpy as np
import pytest
import torch

import ssim_ref as S

pytestmark = pytest.mark.gpu

DEV = "cuda"
SHAPES = [(11, 11), (11, 300), (40, 53), (257, 129), (400, 400), (800, 800), (1021, 37)]
KINDS = ("random", "smooth", "near_constant", "wide")


def _image(kind, H, W, gen):
    r = lambda *s: torch.rand(*s, device=DEV, generator=gen)  # noqa: E731
    if kind == "random":
        x = r(H * W, 3)
        return x, 0.6 * x + 0.4 * r(H * W, 3)
    if kind == "smooth":
        i = torch.arange(H, device=DEV, dtype=torch.float32)[:, None, None] / H
        j = torch.arange(W, device=DEV, dtype=torch.float32)[None, :, None] / W
        c = torch.arange(3, device=DEV, dtype=torch.float32)
        x = (0.5 + 0.4 * torch.sin(2 * np.pi * (1.3 * i + 0.7 * j) + c)).reshape(-1, 3)
        return x, (x + 0.05 * torch.randn(x.shape, device=DEV, generator=gen)).clamp(0, 1)
    if kind == "near_constant":
        return 0.5 + 1e-3 * r(H * W, 3), 0.5 + 1e-3 * r(H * W, 3)
    return r(H * W, 3) * 1.5 - 0.2, r(H * W, 3)


def _batch(H, W, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    pairs = [_image(k, H, W, gen) for k in KINDS]
    return torch.stack([p for p, _ in pairs]), torch.stack([t for _, t in pairs])


@pytest.mark.parametrize("H,W", SHAPES)
def test_ssim_vs_fp64(H, W):
    """B = 4 in one call and each image alone (B = 1): both within the bound, and the same bits."""
    from taichi_nerfs_b200 import ops
    pred, target = _batch(H, W, seed=H * 7 + W)
    got = ops.ssim(pred, target, H, W)
    assert got.shape == (4,) and got.dtype == torch.float32 and got.is_cuda
    singles = torch.cat([ops.ssim(pred[i], target[i], H, W) for i in range(4)])
    assert torch.equal(got.view(torch.int32), singles.view(torch.int32)), (got, singles)
    p, t = pred.cpu().numpy(), target.cpu().numpy()
    worst = S.check(got.cpu().numpy(), p, t, H, W, what=f"{H}x{W}")
    print(f"{H}x{W}: ssim {got.tolist()} fp64 {S.ssim(p, t, H, W).tolist()} worst err/bound {worst:.3g}")


def test_reruns_and_graph_replay_are_bit_identical():
    from taichi_nerfs_b200 import ops
    H, W = 800, 800
    pred, target = _batch(H, W, seed=1)
    eager = ops.ssim(pred, target, H, W)
    for _ in range(3):
        assert torch.equal(ops.ssim(pred, target, H, W).view(torch.int32), eager.view(torch.int32))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        ops.ssim(pred, target, H, W)                 # warm-up on the capture stream
        with torch.cuda.graph(g, stream=s):
            out = ops.ssim(pred, target, H, W)
    torch.cuda.current_stream().wait_stream(s)
    out.fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), eager.view(torch.int32))


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_non_finite_pixel_poisons_only_its_image(bad):
    """A NaN / inf in image 2 of 4 makes its result NaN; the other three are bit-identical to the clean run.  The bad
    pixel sits in the image's last column, which only the last valid window reaches."""
    from taichi_nerfs_b200 import ops
    H, W = 257, 129
    pred, target = _batch(H, W, seed=2)
    clean = ops.ssim(pred, target, H, W)
    p = pred.clone()
    p[1, 100 * W + W - 1, 2] = bad
    got = ops.ssim(p, target, H, W)
    assert bool(torch.isnan(got[1])), got
    keep = [0, 2, 3]
    assert torch.equal(got[keep].view(torch.int32), clean[keep].view(torch.int32))


def test_batch_past_2_pow_31_floats():
    """7200 images of 320 x 320: 2,211,840,000 floats per tensor, so every offset of the last images passes 2^31.
    The first, a middle and the last three images against fp64."""
    from taichi_nerfs_b200 import ops
    B, H, W = 7200, 320, 320
    n = B * H * W * 3
    assert (B - 3) * H * W * 3 > 2 ** 31
    need = 2 * n * 4 + (2 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    pred = target = None
    try:
        gen = torch.Generator(device=DEV).manual_seed(31)
        pred = torch.rand(B, H * W, 3, device=DEV, generator=gen)
        target = torch.rand(B, H * W, 3, device=DEV, generator=gen).mul_(0.4).add_(pred, alpha=0.6)
        for i, kind in zip((B - 3, B - 2, B - 1), ("smooth", "near_constant", "wide")):
            pred[i], target[i] = _image(kind, H, W, gen)
        got = ops.ssim(pred, target, H, W).cpu().numpy()
        idx = [0, B // 2, B - 3, B - 2, B - 1]
        worst = S.check(got[idx], pred[idx].cpu().numpy(), target[idx].cpu().numpy(), H, W, what="B=7200")
        assert np.isfinite(got).all()
        print(f"B=7200 320x320: worst err/bound {worst:.3g}")
    finally:
        del pred, target
        torch.cuda.empty_cache()


def test_train_main_prints_ssim(tmp_path, monkeypatch, capsys):
    import train
    from test_gpu_e2e import _small_dataset
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(train, 'dataset_dict', {'synthetic': _small_dataset})
    psnrs = train.main(['--dataset_name', 'synthetic', '--half_opt', '--batch_size', '4096', '--max_steps', '200'])
    out = capsys.readouterr().out
    m = re.search(r"^evaluation: psnr_avg=(\S+) \| ssim_avg=(\S+)$", out, flags=re.M)
    assert m, out[-2000:]
    assert abs(float(m.group(1)) - sum(psnrs) / len(psnrs)) < 1e-9
    assert 0.0 < float(m.group(2)) <= 1.0, m.group(0)
    print(m.group(0))


def test_train_vs_teacher_reports_ssim():
    """ssim_views of psnr.train_vs_teacher equal the fp64 SSIM of the returned model's re-rendered (clamped) views."""
    import __graft_entry__ as g
    if not g.stage_lego_fixture():
        pytest.skip("shipped Lego weights could not be staged")
    from datasets.ray_utils import get_rays
    from modules.rendering import render
    from taichi_nerfs_b200.psnr import train_vs_teacher
    r = train_vs_teacher(torch.device(DEV), steps=300, train_views=16, test_views=2, downsample=0.25)
    if r is None:
        pytest.skip("teacher fixture not staged")
    assert len(r["ssim_views"]) == len(r["psnr_views"]) == 2
    assert r["ssim"] == sum(r["ssim_views"]) / 2
    model, test_ds = r["model"], r["test_dataset"]
    w, h = test_ds.img_wh
    for i, v in enumerate(r["ssim_views"]):
        td = test_ds[i]
        rays_o, rays_d = get_rays(test_ds.directions, td['pose'])
        with torch.no_grad(), torch.autocast('cuda', dtype=torch.float16):
            res = render(model, rays_o, rays_d, test_time=True)
        pred = res['rgb'].float().clamp(0, 1).cpu().numpy()
        worst = S.check([v], pred, td['rgb'].cpu().numpy(), h, w, what=f"teacher view {i}")
        print(f"teacher view {i}: psnr {r['psnr_views'][i]:.2f} dB ssim {v:.5f} worst err/bound {worst:.3g}")
