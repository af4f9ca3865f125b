"""Depth supervision (--depth_loss_w, DESIGN.md §6h) without a GPU: the flag, the ngp loader's depth_path images and
the batches that carry them, the module-path loss, the fp64 restatement of the fused head's depth term against central
differences, its comparator, and the C-ABI entry's argument checks."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))

from depth_ref import check_head_depth, head_ref_depth  # noqa: E402
from test_gpu_graph_step_distortion import _rays  # noqa: E402

from datasets import dataset_dict  # noqa: E402


# ---- the flag ------------------------------------------------------------------------------------------------------
def test_depth_flag():
    from opt import get_opts
    assert get_opts([]).depth_loss_w == 0
    assert get_opts(['--depth_loss_w', '0.1']).depth_loss_w == 0.1
    assert get_opts(['--dataset_name', 'ngp', '--root_dir', '/x', '--depth_loss_w', '1']).depth_loss_w == 1
    for bad in ('-1e-3', 'nan', 'inf'):
        with pytest.raises(SystemExit):
            get_opts(['--depth_loss_w', bad])
    for name in ('nerf', 'nsvf', 'colmap'):
        with pytest.raises(SystemExit):
            get_opts(['--dataset_name', name, '--root_dir', '/x', '--depth_loss_w', '0.1'])
        assert get_opts(['--dataset_name', name, '--root_dir', '/x']).depth_loss_w == 0


# ---- the ngp loader --------------------------------------------------------------------------------------------------
W, H, SCALE = 8, 6, 0.001


def _ramp(k):
    """A 16-bit depth ramp unique per frame and pixel."""
    return (1000 * (k + 1) + 37 * np.arange(H)[:, None] + 3 * np.arange(W)[None, :]).astype(np.uint16)


def _write_scene(root, depth_size=(W, H), with_scale=True):
    """Frames: 0 and 3 with depth, 1 without depth_path, 2 with depth_path but no image (skipped)."""
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    os.makedirs(os.path.join(root, 'depth'), exist_ok=True)
    rng = np.random.default_rng(0)
    frames = []
    for k in range(4):
        pose = np.eye(4)
        pose[:3, 3] = (0.1 * k, 0.2, 1.5)
        f = {'file_path': f'images/{k}.png', 'transform_matrix': pose.tolist()}
        if k != 2:
            Image.fromarray(rng.integers(0, 255, (H, W, 3), dtype=np.uint8)).save(os.path.join(root, f['file_path']))
        if k != 1:
            f['depth_path'] = f'depth/{k}.png'
            raw = _ramp(k)
            if depth_size != (W, H):
                raw = np.resize(raw, (depth_size[1], depth_size[0]))
            Image.fromarray(raw).save(os.path.join(root, f['depth_path']))
        frames.append(f)
    meta = {'w': W, 'h': H, 'fl_x': 10.0, 'fl_y': 10.0, 'frames': frames}
    if with_scale:
        meta['integer_depth_scale'] = SCALE
    with open(os.path.join(root, 'transforms.json'), 'w') as f:
        json.dump(meta, f)
    return root


def test_ngp_loader_reads_depth(tmp_path):
    root = _write_scene(str(tmp_path / 'scene'))
    assert Image.open(os.path.join(root, 'depth/0.png')).mode.startswith('I')   # a 16-bit single-channel PNG
    d = dataset_dict['ngp'](root, 'train', 1.0)
    assert len(d) == 3 and d.depths.shape == (3, W * H) and d.depths.dtype == torch.float32
    # frames 0, 1, 3: raw x scale, zeros for the frame without depth_path, the skipped frame's depth dropped
    assert np.array_equal(d.depths[0].numpy(), (_ramp(0).astype(np.float64) * SCALE).astype(np.float32).ravel())
    assert not d.depths[1].any()
    assert np.array_equal(d.depths[2].numpy(), (_ramp(3).astype(np.float64) * SCALE).astype(np.float32).ravel())
    assert np.allclose(d.poses[:, 0, 3].numpy(), [0.0, 0.1, 0.3])     # poses keep the same frames
    # --downsample 0.5: 4 x 3, nearest pixels (1, 3, 5, 7) x (1, 3, 5), never an average of two
    h = dataset_dict['ngp'](root, 'train', 0.5)
    assert h.img_wh == (4, 3)
    want = _ramp(3)[1::2, 1::2].astype(np.float64) * SCALE
    assert np.array_equal(h.depths[2].numpy(), want.astype(np.float32).ravel())
    # batches: 'depth' indexed as 'rgb' is
    d.batch_size = 64
    for strategy in ('all_images', 'same_image'):
        d.ray_sampling_strategy = strategy
        s = d[2]
        img = s['img_idxs'] if strategy == 'all_images' else torch.full((64,), 2, dtype=torch.long)
        assert torch.equal(s['depth'], d.depths[img, s['pix_idxs']])
        assert torch.equal(s['rgb'], d.rays[img, s['pix_idxs'], :3])
    t = dataset_dict['ngp'](root, 'test', 1.0)
    assert torch.equal(t[2]['depth'], t.depths[2])


def test_ngp_loader_depth_errors(tmp_path):
    with pytest.raises(ValueError, match='integer_depth_scale'):
        dataset_dict['ngp'](_write_scene(str(tmp_path / 'a'), with_scale=False), 'train', 1.0)
    with pytest.raises(ValueError, match='transforms.json says'):
        dataset_dict['ngp'](_write_scene(str(tmp_path / 'b'), depth_size=(W + 2, H)), 'train', 1.0)
    root = _write_scene(str(tmp_path / 'c'))
    Image.fromarray(np.zeros((H, W, 3), np.uint8)).save(os.path.join(root, 'depth/0.png'))
    with pytest.raises(ValueError, match='single-channel'):
        dataset_dict['ngp'](root, 'train', 1.0)


def test_committed_ngp_fixture_has_no_depth():
    from make_dataset_golden import DATA, case_key
    golden = np.load(os.path.join(ROOT, 'tests', 'golden', 'datasets_golden.npz'))
    d = dataset_dict['ngp'](os.path.join(DATA, 'ngp_scene'), 'train', 0.5)
    assert getattr(d, 'depths', None) is None
    assert np.array_equal(d.rays[..., :3].numpy(), golden[case_key('ngp', 'ngp_scene', 'train') + '__rays'])
    d.batch_size = 16
    torch.manual_seed(4)
    s = d[0]
    assert 'depth' not in s
    torch.manual_seed(4)
    img, pix = torch.randint(0, len(d), (16,)), torch.randint(0, d.img_wh[0] * d.img_wh[1], (16,))
    assert torch.equal(s['img_idxs'], img) and torch.equal(s['pix_idxs'], pix)


# ---- the module path's loss ------------------------------------------------------------------------------------------
def test_depth_loss_module():
    from modules.depth import depth_loss
    D = torch.tensor([1.0, 2.0, 0.5, 0.7, 0.9, 1.1], requires_grad=True)
    gt = torch.tensor([1.5, 0.0, -1.0, float('nan'), float('inf'), 1.0])
    loss = depth_loss({'depth': D}, gt)
    assert torch.allclose(loss, torch.tensor([0.25, 0, 0, 0, 0, 0.01]))
    (0.5 * loss.mean()).backward()
    assert torch.allclose(D.grad, 0.5 * 2 * torch.tensor([-0.5, 0, 0, 0, 0, 0.1]) / 6)
    assert torch.isfinite(D.grad).all()


# ---- the fp64 restatement ----------------------------------------------------------------------------------------------
def _case(seed, half=False):
    """Short rays with a few coarse samples (all active at thr 1e-4), targets of every kind: real, 0, negative, NaN,
    inf, and a ray that misses (0 samples) with a target."""
    rng = np.random.default_rng(seed)
    rays_a, sig, deltas, ts = _rays(rng, [0, 1, 3, 5, 7, 12, 31, 33, 40, 9, 6], 0.0, x_lo=0.02, x_hi=0.2,
                                    d_const=0.05)
    n, S = rays_a.shape[0], sig.size
    rgbs = (rng.random((S, 3)) * 0.8 + 0.1).astype(np.float16 if half else np.float32)
    gt = rng.random((n, 3)).astype(np.float32)
    depth_gt = rng.uniform(0.1, 1.5, n).astype(np.float32)
    depth_gt[rays_a[[1, 2, 3, 4], 0]] = (0.0, -0.5, np.nan, np.inf)
    return (sig, rgbs, deltas, ts, rays_a, gt), depth_gt


@pytest.mark.parametrize("bg_kind", ["const", "colours"])
@pytest.mark.parametrize("w_d", [0.0, 1e-2])
def test_restatement_matches_central_differences(bg_kind, w_d):
    (sig, rgbs, deltas, ts, rays_a, gt), depth_gt = _case(7)
    n = rays_a.shape[0]
    rng = np.random.default_rng(1)
    bg = 1.0 if bg_kind == "const" else (rng.random((n, 3)), rng.random(n), 1.0)
    scale, w_z = 2.0 ** 16, 0.3

    def loss(s):
        return head_ref_depth(s, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, w_z, depth_gt, 1e-4)["loss"] / (3 * n)

    h = head_ref_depth(sig.astype(np.float64), rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, w_z, depth_gt, 1e-4)
    assert h["ref"]["active"].all()
    assert np.count_nonzero(h["v"]) == n - 4 and h["dz"][rays_a[0, 0]] != 0     # the missing ray has a target
    s64 = sig.astype(np.float64)
    for s in np.random.default_rng(2).choice(sig.size, 40, replace=False):
        e = np.zeros(sig.size)
        e[s] = 1e-5 * s64[s]
        fd = (loss(s64 + e) - loss(s64 - e)) / (2 * e[s])
        assert abs(scale * fd - h["ref"]["dsig"][s]) <= 1e-6 * max(abs(h["ref"]["dsig"][s]), 1e-3 * scale), s
    # the depth term is a visible part of those gradients
    h0 = head_ref_depth(s64, rgbs, deltas, ts, rays_a, gt, bg, scale, w_d, 0.0, depth_gt, 1e-4)
    assert np.abs(h["ref"]["dsig"] - h0["ref"]["dsig"]).max() > 1e-2 * np.abs(h0["ref"]["dsig"]).max()
    assert np.array_equal(h["ref"]["drgb"], h0["ref"]["drgb"])                 # no gradient to the colours


def _emulated(case, depth_gt, bg, scale, w_d, w_z, half, faults=()):
    h = head_ref_depth(*case, bg, scale, w_d, w_z, depth_gt, 1e-4, faults=faults)
    return (np.float32(h["loss"]), h["fwd"]["op"].astype(np.float32), h["out"].astype(np.float32),
            h["ref"]["dsig"].astype(np.float32), h["ref"]["drgb"].astype(np.float16 if half else np.float32))


@pytest.mark.parametrize("half", [False, True])
def test_comparator_accepts_the_reference_rounded_to_fp32(half):
    case, depth_gt = _case(11 + half, half)
    for w_d, w_z in ((0.0, 1e-2), (1e-2, 1.0)):
        got = _emulated(case, depth_gt, 1.0, 2.0 ** 16, w_d, w_z, half)
        check_head_depth(got, *case, 1.0, 2.0 ** 16, w_d, w_z, depth_gt, 1e-4, half, "fp64 rounded")


@pytest.mark.parametrize("fault", ["no_gz", "coef_valid", "invalid_as_zero", "bg_in_depth"])
def test_comparator_rejects(fault):
    case, depth_gt = _case(13, True)
    got = _emulated(case, depth_gt, 1.0, 2.0 ** 16, 0.0, 0.1, True, faults=(fault,))
    with pytest.raises(AssertionError):
        check_head_depth(got, *case, 1.0, 2.0 ** 16, 0.0, 0.1, depth_gt, 1e-4, True, fault)


# ---- the C-ABI entry's checks ----------------------------------------------------------------------------------------
def test_depth_entry_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    lib = _lib.load()
    fake = C.c_void_p(0x10000)
    f = lib.ngp_ray_head_fused_depth

    def args(w_z=0.1, w_d=0.0, dgt=fake, ts=fake, bg_rgb=None, alpha=None, dt=1):
        return (fake, fake, dt, fake, ts, fake, fake, 1.0, bg_rgb, alpha, 1.0, 1.0, None, 1e-4, w_d, dgt, w_z, fake,
                None, None, fake, fake, 8, None)
    for w in (-1e-3, float("inf"), float("nan")):
        assert f(*args(w_z=w)) < 0 and b"depth_w" in lib.ngp_last_error()
        assert f(*args(w_d=w)) < 0 and b"distortion_w" in lib.ngp_last_error()
    assert f(*args(dgt=None)) < 0 and b"null" in lib.ngp_last_error()
    assert f(*args(w_z=0.0, dgt=None)) < 0 and b"null" in lib.ngp_last_error()
    assert f(*args(ts=None)) < 0 and b"null" in lib.ngp_last_error()
    assert f(*args(alpha=fake)) < 0 and b"alpha" in lib.ngp_last_error()
    assert f(*args(dt=7)) < 0 and b"dtype" in lib.ngp_last_error()
    assert f(None, None, 1, None, None, None, None, 1.0, None, None, 1.0, 1.0, None, 1e-4, 0.0, None, 0.1, None, None,
             None, None, None, 0, None) == 0
