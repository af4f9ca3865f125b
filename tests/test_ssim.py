"""CPU checks of SSIM (`ngp_ssim`, `ops.ssim`, DESIGN.md §6e): the fp64 restatement tests/ssim_ref.py against an
independent path (scipy's Gaussian filter) and known answers, the C-ABI's argument validation, the refusal of CPU
tensors, and planted mistakes in a numpy fp32 copy of the kernel that the comparator of the GPU tests must reject."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

import ssim_ref as S

SHAPES = [(11, 11), (11, 300), (40, 53), (257, 129)]


def _content(kind, H, W, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        x = rng.random((H * W, 3))
        return x, 0.6 * x + 0.4 * rng.random((H * W, 3))
    if kind == "smooth":
        i, j = np.meshgrid(np.arange(H) / H, np.arange(W) / W, indexing="ij")
        x = np.stack([0.5 + 0.4 * np.sin(2 * np.pi * (1.3 * i + 0.7 * j) + c) for c in range(3)], -1).reshape(-1, 3)
        return x, np.clip(x + 0.05 * rng.standard_normal(x.shape), 0, 1)
    # near-constant: C2 dominates the variance term
    return 0.5 + 1e-3 * rng.random((H * W, 3)), 0.5 + 1e-3 * rng.random((H * W, 3))


def _scipy_ssim(pred, target, H, W):
    """The moments from scipy's Gaussian filter (sigma 1.5, radius int(truncate * sigma + 0.5) = 5, so the same
    normalised 11-tap window), cropped by 5 on each side to the valid positions."""
    x, y = S.images(pred, H, W)[0], S.images(target, H, W)[0]

    def f(a):
        return np.stack([gaussian_filter(c, 1.5, truncate=5 / 1.5)[5:-5, 5:-5] for c in a])

    return S.ssim_map(f(x), f(y), f(x * x), f(y * y), f(x * y)).mean()


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("kind", ["random", "smooth", "near_constant"])
def test_reference_matches_scipy_gaussian_filter(H, W, kind):
    x, y = _content(kind, H, W, seed=H * 1000 + W)
    ref = S.ssim(x, y, H, W)
    assert ref.shape == (1,)
    assert abs(ref[0] - _scipy_ssim(x, y, H, W)) <= 1e-12, (ref[0], _scipy_ssim(x, y, H, W))


def test_window():
    g = S.window()
    assert len(g) == 11 and abs(g.sum() - 1) < 1e-15 and np.allclose(g, g[::-1], rtol=0, atol=0)
    # torchmetrics' size int(3.5 sigma + 0.5) * 2 + 1 for sigma = 1.5
    assert int(3.5 * 1.5 + 0.5) * 2 + 1 == 11


def test_known_answers():
    rng = np.random.default_rng(3)
    x = rng.random((40 * 53, 3))
    assert abs(S.ssim(x, x, 40, 53)[0] - 1.0) < 1e-14
    a, b = np.full((40 * 53, 3), 0.5), np.full((40 * 53, 3), 0.25)
    want = (2 * 0.5 * 0.25 + S.C1) / (0.5 ** 2 + 0.25 ** 2 + S.C1)
    assert abs(want - 0.2501 / 0.3126) < 1e-15 and abs(want - 0.8000639795) < 1e-10
    assert abs(S.ssim(a, b, 40, 53)[0] - want) < 1e-12
    assert abs(S.kernel_np(a, b, 40, 53)[0] - want) < 1e-6
    y = np.clip(x + 0.1 * rng.standard_normal(x.shape), 0, 1)
    assert S.ssim(x, y, 40, 53)[0] == S.ssim(y, x, 40, 53)[0]       # symmetric in its arguments


def test_single_window_at_11x11():
    rng = np.random.default_rng(11)
    x, y = rng.random((121, 3)), rng.random((121, 3))
    mx, my, exx, eyy, exy = S.moments(S.images(x, 11, 11), S.images(y, 11, 11))
    assert mx.shape == (1, 3, 1, 1)                                   # one position per channel
    G = np.outer(S.window(), S.window())
    xs, ys = S.images(x, 11, 11)[0], S.images(y, 11, 11)[0]
    direct = [S.ssim_map((G * a).sum(), (G * b).sum(), (G * a * a).sum(), (G * b * b).sum(), (G * a * b).sum())
              for a, b in zip(xs, ys)]
    assert abs(S.ssim(x, y, 11, 11)[0] - np.mean(direct)) < 1e-14


def test_batch_is_per_image():
    rng = np.random.default_rng(5)
    x, y = rng.random((3, 40 * 53, 3)), rng.random((3, 40 * 53, 3))
    both = S.ssim(x, y, 40, 53)
    assert both.shape == (3,)
    for i in range(3):
        assert both[i] == S.ssim(x[i], y[i], 40, 53)[0]


def test_cabi_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib
    L = _lib.load()
    p = C.c_void_p(16)

    def call(n=2, h=40, w=53, ptrs=(p, p, p, p)):
        return L.ngp_ssim(ptrs[0], ptrs[1], n, h, w, ptrs[2], ptrs[3], None)

    for i in range(4):
        ptrs = [p] * 4
        ptrs[i] = None
        assert call(ptrs=tuple(ptrs)) < 0
        assert b"null" in L.ngp_last_error()
    for h, w in ((10, 53), (40, 10), (0, 0), (-5, 40)):
        assert call(h=h, w=w) < 0
        assert b"11" in L.ngp_last_error()
    assert call(n=-1) < 0 and b"negative" in L.ngp_last_error()
    assert call(n=0, ptrs=(None,) * 4) == 0                          # no images: a no-op
    assert call(n=2 ** 40) < 0 and b"too many" in L.ngp_last_error()


def test_ops_refuses_cpu_tensors():
    from taichi_nerfs_b200 import _lib, ops
    x = torch.rand(40 * 53, 3)
    with pytest.raises(_lib.NgpError):
        ops.ssim(x, x, 40, 53)
    with pytest.raises(_lib.NgpError):
        ops.ssim(x.unsqueeze(0), x.unsqueeze(0), 40, 53)


# ---- fault injection for the comparator ---------------------------------------------------------------------------
def _blocks(H, W, seed):
    """Piecewise-constant 4x4-pixel blocks and the same image shifted by one pixel: the window's shape matters."""
    rng = np.random.default_rng(seed)
    x = np.repeat(np.repeat(rng.random((H // 4 + 1, W // 4 + 2, 3)), 4, 0), 4, 1)
    return x[:H, 1:W + 1].reshape(-1, 3), x[:H, :W].reshape(-1, 3)


def _fault_case():
    """Random, smooth and blocky content (a 10-tap window barely moves the SSIM of i.i.d. noise; the blocks catch it)."""
    cases = [_content("random", 40, 53, seed=9), _content("smooth", 40, 53, seed=10), _blocks(40, 53, seed=11)]
    return tuple(np.stack([c[k] for c in cases]).astype(np.float32) for k in (0, 1))


def test_comparator_accepts_numpy_fp32_copy():
    x, y = _fault_case()
    worst = S.check(S.kernel_np(x, y, 40, 53), x, y, 40, 53, what="numpy fp32")
    assert 0 <= worst <= 1
    for kind in ("random", "smooth", "near_constant"):
        for H, W in SHAPES:
            a, b = (v.astype(np.float32) for v in _content(kind, H, W, seed=1))
            S.check(S.kernel_np(a, b, H, W), a, b, H, W, what=f"numpy fp32 {kind} {H}x{W}")


@pytest.mark.parametrize("fault", S.FAULTS)
def test_comparator_rejects_planted_mistakes(fault):
    x, y = _fault_case()
    with pytest.raises(AssertionError, match="off the fp64 bound"):
        S.check(S.kernel_np(x, y, 40, 53, fault=fault), x, y, 40, 53, what=f"numpy fault={fault}")
    with pytest.raises(AssertionError, match="off the fp64 bound"):       # the blocky image alone
        S.check(S.kernel_np(x[2], y[2], 40, 53, fault=fault), x[2], y[2], 40, 53, what=f"numpy fault={fault}")
