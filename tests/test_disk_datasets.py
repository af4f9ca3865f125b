"""The reference's disk loaders (datasets/{nerf,nsvf,ngp,colmap}.py) on the tiny fixtures under tests/golden/datasets/:
bit-identical to the reference's outputs stored in tests/golden/datasets_golden.npz (tests/golden/make_dataset_golden.py
wrote both), batch sampling, the COLMAP binary reader, image validation and the command-line flags."""
import json
import os
import shutil
import struct
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
sys.path.insert(0, GOLDEN)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from colmap_writer import cameras_bytes, images_bytes, points_bytes, rotmat2qvec, write_model  # noqa: E402
from make_dataset_golden import CASES, DATA, case_key  # noqa: E402

from datasets import dataset_dict  # noqa: E402
from datasets import colmap_model as CM  # noqa: E402
from datasets.color_utils import read_image  # noqa: E402


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(GOLDEN, 'datasets_golden.npz')))


@pytest.mark.parametrize('name,root,split,down', CASES, ids=[case_key(*c[:3]) for c in CASES])
def test_loader_matches_reference(golden, name, root, split, down):
    d = dataset_dict[name](root_dir=os.path.join(DATA, root), split=split, downsample=down)
    key = case_key(name, root, split)
    assert d.K.dtype == d.poses.dtype == d.directions.dtype == torch.float32
    assert np.array_equal(d.K.numpy(), golden[key + '__K'])
    assert tuple(d.img_wh) == tuple(golden[key + '__img_wh'])
    assert np.array_equal(d.directions.numpy(), golden[key + '__directions'])
    assert d.poses.shape[1:] == (3, 4)
    assert np.array_equal(d.poses.numpy(), golden[key + '__poses'])
    ref_rays = golden[key + '__rays']
    if ref_rays.size == 0:
        assert len(d.rays) == 0
        return
    assert d.rays.dtype == torch.float32
    assert np.array_equal(d.rays[..., :3].numpy(), ref_rays)
    if key + '__alpha' in golden:
        assert d.rays.shape[-1] == 4
        assert np.array_equal(d.rays[..., 3].numpy(), golden[key + '__alpha'])
    else:
        assert d.rays.shape[-1] == 3


def test_fixture_branches():
    """The name-dependent branches the fixtures exercise are the ones meant."""
    nsvf = dataset_dict['nsvf'](os.path.join(DATA, 'Synthetic_NeRF/Lego'), 'train', 0.02)
    lo = np.array([-0.637787, -1.140016, -0.344656])
    hi = np.array([0.633744, 1.148737, 1.002206])
    assert nsvf.scale == (hi - lo).max() / 2 * 1.05 * 1.1          # the Lego correction
    assert np.allclose(nsvf.shift, (hi + lo) / 2)
    col = dataset_dict['colmap'](os.path.join(DATA, '360_v2/garden'), 'test', 0.25)
    assert col.img_wh == (16, 12) and len(col) == 2             # images_4/ at downsample 0.25, every 8th of ten
    every = dataset_dict['colmap'](os.path.join(DATA, '360_v2/garden'), 'trainval', 0.25)
    assert len(every) == 10                                     # a split other than train/test reads every image
    assert np.isclose(np.linalg.norm(every.poses[:, :, 3].numpy(), axis=-1).min(), 1.0, atol=1e-6)  # nearest at 1
    ngp = dataset_dict['ngp'](os.path.join(DATA, 'ngp_scene'), 'train', 0.5)
    assert len(ngp) == 3                                          # the frame without an image file is skipped


@pytest.mark.parametrize('strategy', ['all_images', 'same_image'])
def test_sampling(strategy):
    d = dataset_dict['nerf'](os.path.join(DATA, 'nerf_blender'), 'train', 0.02)
    d.batch_size, d.ray_sampling_strategy = 64, strategy
    torch.manual_seed(3)
    s = d[1]
    torch.manual_seed(3)
    if strategy == 'all_images':
        img = torch.randint(0, len(d.poses), (64,))
    else:
        img = torch.full((64,), 1, dtype=torch.long)
    pix = torch.randint(0, 16 * 16, (64,))
    assert torch.equal(s['pix_idxs'], pix)
    assert torch.equal(s['rgb'], d.rays[img, pix, :3])
    assert torch.equal(s['alpha'], d.rays[img, pix, 3])
    assert torch.equal(s['direction'], d.directions[pix])
    assert s['pose'].shape[-2:] == (3, 4)
    assert torch.equal(s['pose'].expand(64, 3, 4), d.poses[img])
    if strategy == 'all_images':
        assert torch.equal(s['img_idxs'], img)


def test_test_split_items():
    d = dataset_dict['colmap'](os.path.join(DATA, '360_v2/garden'), 'test', 0.25)
    s = d[1]
    assert s['img_idxs'] == 1 and torch.equal(s['pose'], d.poses[1]) and torch.equal(s['rgb'], d.rays[1])
    assert 'alpha' not in s
    t = dataset_dict['nsvf'](os.path.join(DATA, 'Synthetic_NeRF/Lego'), 'test_traj', 0.02)
    assert len(t) == 4 and set(t[0]) == {'pose', 'img_idxs'}
    n = dataset_dict['nerf'](os.path.join(DATA, 'nerf_blender'), 'test', 0.02)
    assert torch.equal(n[0]['alpha'], n.rays[0, :, 3])


def test_colmap_test_traj_poses():
    from datasets.ray_utils import create_spheric_poses
    p = create_spheric_poses(1.2, 0.3, n_poses=6)
    assert p.shape == (6, 3, 4)
    assert np.allclose(p[:, :, :3] @ p[:, :, :3].transpose(0, 2, 1), np.eye(3))


def _model(tmp_path, cam_model, params):
    R = np.linalg.qr(np.random.default_rng(0).normal(size=(3, 3)))[0]
    R *= np.sign(np.linalg.det(R))
    imgs = [(4, rotmat2qvec(R), np.array([0.1, -0.2, 0.3]), 1, 'b.png', np.array([[1.5, 2.5]]), np.array([-1])),
            (2, rotmat2qvec(R.T), np.array([1.0, 2.0, 3.0]), 1, 'a.png', np.zeros((0, 2)), np.zeros(0, np.int64))]
    pts = [(9, np.array([0.5, 0.25, -1.0]), np.array([1, 2, 3]), 0.75, [4, 2], [0, 7])]
    sparse = tmp_path / 'sparse' / '0'
    write_model(str(sparse), [(1, cam_model, 40, 30, params)], imgs, pts)
    return sparse, R, imgs


@pytest.mark.parametrize('model,params', [('SIMPLE_RADIAL', [30.0, 20.0, 15.0, 0.01]),
                                          ('PINHOLE', [30.0, 31.0, 20.0, 15.0]),
                                          ('OPENCV', [30.0, 31.0, 20.0, 15.0, 0.1, 0.2, 0.01, 0.02])])
def test_colmap_reader_round_trip(tmp_path, model, params):
    sparse, R, imgs = _model(tmp_path, model, params)
    cams = CM.read_cameras_binary(str(sparse / 'cameras.bin'))
    assert list(cams) == [1] and cams[1].model == model and (cams[1].width, cams[1].height) == (40, 30)
    assert np.array_equal(cams[1].params, params)
    ims = CM.read_images_binary(str(sparse / 'images.bin'))
    assert list(ims) == [4, 2] and [i.name for i in ims.values()] == ['b.png', 'a.png']
    assert np.allclose(ims[4].qvec2rotmat(), R) and np.allclose(ims[2].qvec2rotmat(), R.T)
    assert np.array_equal(ims[4].tvec, [0.1, -0.2, 0.3])
    assert np.array_equal(ims[4].xys, [[1.5, 2.5]]) and list(ims[4].point3D_ids) == [-1]
    assert ims[2].xys.shape == (0, 2)
    pts = CM.read_points3d_binary(str(sparse / 'points3D.bin'))
    assert list(pts) == [9] and np.array_equal(pts[9].xyz, [0.5, 0.25, -1.0]) and list(pts[9].rgb) == [1, 2, 3]
    assert pts[9].error == 0.75 and list(pts[9].image_ids) == [4, 2] and list(pts[9].point2D_idxs) == [0, 7]
    # the loader takes camera 1's intrinsics as the reference does
    (tmp_path / 'images').mkdir()
    d = dataset_dict['colmap'](str(tmp_path), 'train', 1.0, read_meta=False)
    f = params[0]
    fy, cx, cy = (f, params[1], params[2]) if model == 'SIMPLE_RADIAL' else params[1:4]
    assert np.array_equal(d.K.numpy(), np.float32([[f, 0, cx], [0, fy, cy], [0, 0, 1]]))


@pytest.mark.parametrize('name', ['cameras.bin', 'images.bin', 'points3D.bin'])
def test_colmap_reader_truncated(tmp_path, name):
    sparse, _, _ = _model(tmp_path, 'PINHOLE', [30.0, 31.0, 20.0, 15.0])
    reader = {'cameras.bin': CM.read_cameras_binary, 'images.bin': CM.read_images_binary,
              'points3D.bin': CM.read_points3d_binary}[name]
    raw = (sparse / name).read_bytes()
    for cut in (1, 7, 9, len(raw) // 2, len(raw) - 1):
        (sparse / name).write_bytes(raw[:cut])
        with pytest.raises(ValueError):
            reader(str(sparse / name))
    (sparse / name).write_bytes(raw + b'\0')
    with pytest.raises(ValueError, match='trailing'):
        reader(str(sparse / name))
    # a count far beyond the file
    (sparse / name).write_bytes(struct.pack('<Q', 1 << 60) + raw[8:])
    with pytest.raises(ValueError, match='truncated'):
        reader(str(sparse / name))


def test_colmap_camera_models_refused(tmp_path):
    sparse, _, _ = _model(tmp_path, 'SIMPLE_PINHOLE', [30.0, 20.0, 15.0])
    with pytest.raises(ValueError, match='SIMPLE_PINHOLE'):
        dataset_dict['colmap'](str(tmp_path), 'train', 1.0)
    (sparse / 'cameras.bin').write_bytes(cameras_bytes([(1, 42, 40, 30, [1.0, 2.0, 3.0])]))
    with pytest.raises(ValueError, match='model id 42'):
        CM.read_cameras_binary(str(sparse / 'cameras.bin'))
    with pytest.raises(ValueError, match='HDR-NeRF'):
        dataset_dict['colmap'](str(tmp_path / 'HDR-NeRF' / 'x'), 'train', 1.0)
    assert images_bytes([]) == points_bytes([]) == struct.pack('<Q', 0)


def _png(path, arr, mode=None):
    from PIL import Image
    Image.fromarray(arr, mode=mode).save(path) if mode else Image.fromarray(arr).save(path)


def test_read_image_refuses_bad_images(tmp_path):
    from PIL import Image
    gray = tmp_path / 'gray.png'
    Image.fromarray(np.full((4, 4), 7, np.uint8)).save(gray)
    with pytest.raises(ValueError, match="mode 'L'"):
        read_image(str(gray), (4, 4))
    g16 = tmp_path / 'g16.png'
    Image.fromarray(np.full((4, 4), 40000, np.uint16)).save(g16)
    with pytest.raises(ValueError):
        read_image(str(g16), (4, 4))
    # 16-bit RGB: PIL would hand back 8 bits; the IHDR bit depth is checked instead
    import zlib
    raw = b''.join(b'\0' + np.full((4, 3), 0x1234, '>u2').tobytes() for _ in range(4))

    def chunk(t, d):
        return struct.pack('>I', len(d)) + t + d + struct.pack('>I', zlib.crc32(t + d))
    png = (b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', 4, 4, 16, 2, 0, 0, 0))
           + chunk(b'IDAT', zlib.compress(raw)) + chunk(b'IEND', b''))
    (tmp_path / 'rgb16.png').write_bytes(png)
    with pytest.raises(ValueError, match='16-bit'):
        read_image(str(tmp_path / 'rgb16.png'), (4, 4))


def test_read_image_blending(tmp_path):
    rgba = np.random.default_rng(1).integers(0, 256, (6, 5, 4), dtype=np.uint8)
    _png(tmp_path / 'a.png', rgba)
    f = rgba.astype(np.float32) / 255.0
    white = read_image(str(tmp_path / 'a.png'), (5, 6))
    assert np.array_equal(white, (f[..., :3] * f[..., 3:] + (1 - f[..., 3:])).reshape(-1, 3))
    black = read_image(str(tmp_path / 'a.png'), (5, 6), blend_a=False, keep_alpha=True)
    assert np.array_equal(black, np.concatenate([f[..., :3] * f[..., 3:], f[..., 3:]], -1).reshape(-1, 4))
    _png(tmp_path / 'b.png', rgba[..., :3])
    assert read_image(str(tmp_path / 'b.png'), (5, 6), keep_alpha=True).shape == (30, 3)


def test_mixed_alpha_and_jade(tmp_path):
    """Images with and without alpha in one split: alpha 1 for the opaque ones.  Jade/Fountain: dark pixels -> 1."""
    src = os.path.join(DATA, 'Synthetic_NeRF', 'Lego')
    dst = tmp_path / 'BlendedMVS' / 'Jade'
    shutil.copytree(src, dst)
    np.savetxt(dst / 'intrinsics.txt', np.array([[20.0, 0, 8], [0, 20.0, 6], [0, 0, 1]]))
    img = np.full((576, 768, 3), 200, np.uint8)
    img[:100, :100] = 10
    _png(dst / 'rgb' / '0_0001.png', img)
    d = dataset_dict['nsvf'](str(dst), 'train', 0.02)
    assert d.img_wh == (15, 11) and d.rays.shape == (3, 165, 4)
    assert torch.all(d.rays[1, :, 3] == 1.0)
    assert torch.all(d.rays[1, 0, :3] == 1.0)                     # dark corner pixel -> white
    assert torch.all(torch.isclose(d.rays[1, -1, :3], torch.tensor(200 / 255.0)))


def test_nsvf_unknown_directory(tmp_path):
    shutil.copytree(os.path.join(DATA, 'Synthetic_NeRF', 'Lego'), tmp_path / 'Scene')
    with pytest.raises(ValueError, match='Synthetic, Ignatius, BlendedMVS or Tanks'):
        dataset_dict['nsvf'](str(tmp_path / 'Scene'), 'train', 0.02)


def test_nerf_frame_without_image(tmp_path):
    """A held-out frame without its image keeps its pose (as in the reference); a training split refuses it."""
    dst = tmp_path / 'blender'
    shutil.copytree(os.path.join(DATA, 'nerf_blender'), dst)
    os.remove(dst / 'test' / 'r_1.png')
    d = dataset_dict['nerf'](str(dst), 'test', 0.02)
    assert len(d.poses) == 2 and len(d.rays) == 1
    with open(dst / 'transforms_test.json') as f:
        assert len(json.load(f)['frames']) == 2
    os.remove(dst / 'train' / 'r_2.png')
    for split in ('train', 'trainval'):
        with pytest.raises(ValueError, match='1 of the'):
            dataset_dict['nerf'](str(dst), split, 0.02)


def test_opts():
    from opt import get_opts
    for name in ('nerf', 'nsvf', 'colmap', 'ngp'):
        h = get_opts(['--dataset_name', name, '--root_dir', '/data/x'])
        assert h.dataset_name == name and h.root_dir == '/data/x'
        with pytest.raises(SystemExit):
            get_opts(['--dataset_name', name])
    assert get_opts(['--random_bg']).random_bg
    assert get_opts([]).dataset_name == 'synthetic'


def test_gui_camera_takes_disk_poses():
    from gui import OrbitCamera
    d = dataset_dict['colmap'](os.path.join(DATA, '360_v2/garden'), 'train', 0.25)
    cam = OrbitCamera(d.K, d.img_wh, d.poses, r=2.0)
    assert np.allclose(cam.rot, d.poses[0, :, :3].numpy()) and cam.pose.shape == (4, 4)
