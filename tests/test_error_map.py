"""CPU checks of error-map sampling (DESIGN.md §6j): flag validation, the integer restatement's own properties (tile
mapping, rebuild bounds, uniform weights of exactly 1, the 1/alpha weight bound) and ``gather`` of the datasets."""
import numpy as np
import pytest
import torch

import error_map_ref as R


# ---- flags ---------------------------------------------------------------------------------------------------------
def test_error_map_flag_needs_one_rank(monkeypatch):
    from opt import get_opts
    assert get_opts(['--ray_sampling_strategy', 'error_map']).ray_sampling_strategy == 'error_map'
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit):
        get_opts(['--ray_sampling_strategy', 'error_map'])
    assert get_opts([]).ray_sampling_strategy == 'all_images'   # other strategies keep running on several ranks


@pytest.mark.parametrize("res", ["0", "-3", "4097"])
def test_error_map_res_validated(res):
    from opt import get_opts
    with pytest.raises(SystemExit):
        get_opts(['--ray_sampling_strategy', 'error_map', '--error_map_res', res])


def test_floor_fraction():
    from taichi_nerfs_b200.error_map import floor_fraction
    assert floor_fraction(0.2) == (1, 5)
    assert floor_fraction(0.5) == (1, 2)
    for bad in (0.0, 1.0, -0.1, 2.0):
        with pytest.raises(ValueError):
            floor_fraction(bad)


def test_kernel_arguments_validated_without_gpu():
    """Bad geometry, floors and sizes are refused (rc < 0) before any launch."""
    from taichi_nerfs_b200 import _lib, build
    build.build()
    L = _lib.load()
    assert L.ngp_error_map_workspace_bytes(1) == 8 * 9
    assert L.ngp_error_map_sample(None, 1, 4, 4, 5, 0, None, 0, None, None, None, 8, None) < 0      # R > min(W, H)
    assert L.ngp_error_map_sample(None, 1 << 20, 1 << 10, 1 << 10, 1, 0, None, 0, None, None, None, 8, None) < 0
    assert L.ngp_error_map_sample(None, 1, 4, 4, 2, 0, None, 0, None, None, None, 8, None) < 0       # null
    assert L.ngp_error_map_sample(None, 1, 4, 4, 2, 0, None, 0, None, None, None, 0, None) == 0      # empty
    assert L.ngp_error_map_accumulate(None, None, None, None, 1.0, None, None, 1, 4, 4, 2, None, None, 4, None) < 0
    for sh, p, q in ((32, 1, 5), (2, 0, 5), (2, 5, 5), (2, 1, 2048)):
        assert L.ngp_error_map_rebuild(None, None, None, None, 1, 4, 4, 2, sh, p, q, None, 0, None) < 0
    assert L.ngp_ray_grad_weight(None, None, None, None, 7, None, 4, 4, None) < 0                       # dtype
    assert L.ngp_ray_grad_weight(None, None, None, None, 0, None, 0, 4, None) == 0


# ---- the restatement -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", [(1, 1, 1, 1), (2, 7, 5, 3), (3, 100, 75, 64), (1, 64, 64, 64), (2, 130, 97, 13)])
def test_tiles_partition_every_image(geom):
    n_img, W, H, Rr = geom
    n_t = R.tile_pixels(geom)
    assert n_t.shape == (n_img * Rr * Rr,) and n_t.min() >= 1 and n_t.sum() == n_img * W * H
    img = np.repeat(np.arange(n_img), W * H)
    pix = np.tile(np.arange(W * H), n_img)
    counts = np.bincount(R.tile_of(img, pix, geom), minlength=len(n_t))
    np.testing.assert_array_equal(counts, n_t)
    # out-of-range indices are clamped as the batch sampler clamps them
    assert R.tile_of([-5, n_img + 3], [-1, W * H + 9], geom).tolist() == [0, len(n_t) - 1]


def test_errors_fixed_point():
    pred = np.array([[0.5, 0.5, 0.5], [1, 1, 1], [0, 0, 0], [np.nan, 0, 0], [0.25, 0, 0]], np.float32)
    tgt = np.array([[0.5, 0.5, 0.5], [0, 0, 0], [1, 1, 1], [0, 0, 0], [0, 0, 0]], np.float32)
    u = R.errors_u(pred, tgt)
    assert u.tolist() == [0, 3 * R.FIX, 3 * R.FIX, 3 * R.FIX, R.FIX // 16]


def test_uniform_map_weights_are_one():
    geom = (5, 123, 77, 64)
    T = 5 * 64 * 64
    for e0 in (0, 1, 12345, 3 * R.FIX):
        E, cdf, info = R.rebuild(np.full(T, e0, np.int64), np.zeros(T, np.int64), np.zeros(T, np.int64), geom)
        assert info["M"] == info["c"] * 5 * 123 * 77 + info["S"]
        img, pix, w = R.sample(cdf, geom, seed=7, step=3, n=20000)
        assert (w == np.float32(1.0)).all()
        assert img.min() >= 0 and img.max() < 5 and pix.min() >= 0 and pix.max() < 123 * 77


@pytest.mark.parametrize("p,q", [(1, 5), (1, 2), (1, 10), (3, 7)])
def test_skewed_map_weights_bounded(p, q):
    geom = (4, 90, 60, 16)
    T = 4 * 16 * 16
    rng = np.random.default_rng(1)
    E = np.zeros(T, np.int64)
    E[rng.integers(0, T, 5)] = 3 * R.FIX     # a few tiles with the largest error, the rest none
    _, cdf, info = R.rebuild(E, np.zeros(T, np.int64), np.zeros(T, np.int64), geom, p=p, q=q)
    img, pix, w = R.sample(cdf, geom, seed=11, step=0, n=50000)
    assert w.max() <= np.float32(q / p) and w.min() > 0
    # every pixel keeps probability >= alpha / N_pix: the smallest mass per pixel is c, and c N_pix >= alpha M
    assert info["c"] * 4 * 90 * 60 * q >= p * info["M"]


def test_rebuild_ema_and_clear():
    geom = (1, 8, 8, 2)
    E = np.array([100, 100, 100, 7], np.int64)
    acc = np.array([400, 0, 50, 1], np.int64)
    cnt = np.array([2, 0, 1, 1], np.int64)
    E2, _, _ = R.rebuild(E, acc, cnt, geom, ema_shift=2)
    # (200-100)>>2 = 25; unseen keeps 100; (50-100)>>2 = -13 (floor); (1-7)>>2 = -2
    assert E2.tolist() == [125, 100, 87, 5]
    assert not acc.any() and not cnt.any()


def test_rebuild_shift_keeps_cdf_below_2_53():
    geom = (64, 4096, 4096, 64)     # N_pix = 2^30: the largest errors need a shift
    T = 64 * 64 * 64
    E = np.full(T, 3 * R.FIX, np.int64)
    E[::7] = 0
    _, cdf, info = R.rebuild(E, np.zeros(T, np.int64), np.zeros(T, np.int64), geom)
    assert info["k"] > 0 and (info["emax"] >> info["k"]) <= info["lim"] < (info["emax"] >> (info["k"] - 1))
    assert int(cdf[-1]) < (1 << 53)


# ---- datasets ------------------------------------------------------------------------------------------------------
def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        torch.testing.assert_close(torch.as_tensor(a[k]), torch.as_tensor(b[k]), rtol=0, atol=0)


def test_base_dataset_gather_equals_getitem():
    from datasets.base import BaseDataset
    ds = BaseDataset('', split='train')
    ds.img_wh = (6, 4)
    g = torch.Generator().manual_seed(0)
    ds.rays = torch.rand(3, 24, 4, generator=g)   # with an alpha column
    ds.depths = torch.rand(3, 24, generator=g)
    ds.poses = torch.rand(3, 3, 4, generator=g)
    ds.directions = torch.rand(24, 3, generator=g)
    ds.batch_size = 50
    for strategy in ('all_images', 'same_image'):
        ds.ray_sampling_strategy = strategy
        s = ds[1]
        assert 'alpha' in s and 'depth' in s
        _same(s, ds.gather(s['img_idxs'], s['pix_idxs']))


def test_synthetic_and_teacher_gather_equal_getitem():
    from datasets.synthetic import SyntheticLego
    from datasets.teacher import TeacherLego
    ds = SyntheticLego(n_images=3, downsample=0.02, batch_size=64, scene='analytic', with_depth=True)
    s = ds[0]
    _same(s, ds.gather(s['img_idxs'], s['pix_idxs']))
    t = TeacherLego(n_images=3, downsample=0.02, batch_size=64)
    t.images = torch.rand(3, t.img_wh[0] * t.img_wh[1], 3)
    s = t[2]
    _same(s, t.gather(s['img_idxs'], s['pix_idxs']))
