"""Camera intrinsics (--lens_distortion, --intrinsics_lr, DESIGN.md §6l) without a GPU: the options' refusals, the
loaders' cameras (and that nothing changes without the flag), the fp64 restatement of the distortion map, its inverse
and its Jacobian, and the C-ABI argument checks of the three new entries."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import camera_ref as ref
from colmap_writer import rotmat2qvec, write_model


# ---- opt.py ---------------------------------------------------------------------------------------------------------
def _opts(*args):
    from opt import get_opts
    return get_opts(list(args))


def test_defaults_leave_hparams_as_before():
    h = _opts()
    assert h.lens_distortion is False and h.intrinsics_lr == 0.0
    assert _opts('--intrinsics_lr', '1e-3').intrinsics_lr == 1e-3
    assert _opts('--dataset_name', 'colmap', '--root_dir', 'x', '--lens_distortion').lens_distortion is True


@pytest.mark.parametrize("v", ["-1e-3", "nan", "inf"])
def test_intrinsics_lr_must_be_finite_and_non_negative(v, capsys):
    with pytest.raises(SystemExit):
        _opts(f'--intrinsics_lr={v}')
    assert "--intrinsics_lr must be finite and >= 0" in capsys.readouterr().err


@pytest.mark.parametrize("flags, what", [(('--model_name', 'svox'), "svox"),
                                         (('--encoder_type', 'triplane'), "triplane"),
                                         (('--lr', '0'), "finite --lr > 0"),
                                         (('--lr', 'nan'), "finite --lr > 0")])
def test_intrinsics_lr_refusals(flags, what, capsys):
    with pytest.raises(SystemExit):
        _opts('--intrinsics_lr', '1e-3', *flags)
    assert what in capsys.readouterr().err


def test_intrinsics_lr_refuses_several_ranks(monkeypatch, capsys):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit):
        _opts('--intrinsics_lr', '1e-3')
    assert "one GPU" in capsys.readouterr().err


@pytest.mark.parametrize("name", ["synthetic", "teacher", "nerf", "nsvf"])
def test_lens_distortion_needs_colmap_or_ngp(name, capsys):
    args = ['--dataset_name', name, '--lens_distortion'] + (['--root_dir', 'x'] if name in ('nerf', 'nsvf') else [])
    with pytest.raises(SystemExit):
        _opts(*args)
    assert "--lens_distortion" in capsys.readouterr().err


def test_intrinsics_combines_with_the_other_refinements():
    h = _opts('--intrinsics_lr', '1e-3', '--extrinsics_lr', '1e-3', '--exposure_lr', '1e-3', '--dataset_name',
              'teacher', '--ray_sampling_strategy', 'error_map', '--distortion_loss_w', '1e-3', '--random_bg')
    assert h.intrinsics_lr == 1e-3


# ---- loaders --------------------------------------------------------------------------------------------------------
def _colmap(tmp_path, cam_model, params, W=40, H=30):
    R = np.eye(3)
    imgs = [(1, rotmat2qvec(R), np.array([0.1, -0.2, 0.3]), 1, 'a.png', np.zeros((0, 2)), np.zeros(0, np.int64))]
    pts = [(9, np.array([0.5, 0.25, -1.0]), np.array([1, 2, 3]), 0.75, [1], [0])]
    write_model(str(tmp_path / 'sparse' / '0'), [(1, cam_model, W, H, params)], imgs, pts)
    (tmp_path / 'images').mkdir(exist_ok=True)
    return str(tmp_path)


@pytest.mark.parametrize('model,params,want', [
    ('SIMPLE_RADIAL', [30.0, 20.0, 15.0, -0.1], (30.0, 30.0, 20.0, 15.0, (-0.1, 0.0, 0.0, 0.0))),
    ('RADIAL', [30.0, 20.0, 15.0, -0.1, 0.02], (30.0, 30.0, 20.0, 15.0, (-0.1, 0.02, 0.0, 0.0))),
    ('OPENCV', [30.0, 31.0, 20.0, 15.0, 0.1, 0.2, 0.01, 0.02], (30.0, 31.0, 20.0, 15.0, (0.1, 0.2, 0.01, 0.02))),
    ('PINHOLE', [30.0, 31.0, 20.0, 15.0], (30.0, 31.0, 20.0, 15.0, (0.0, 0.0, 0.0, 0.0))),
    ('SIMPLE_PINHOLE', [30.0, 20.0, 15.0], (30.0, 30.0, 20.0, 15.0, (0.0, 0.0, 0.0, 0.0)))])
def test_colmap_camera(tmp_path, model, params, want):
    from datasets import dataset_dict
    root = _colmap(tmp_path, model, params)
    d = dataset_dict['colmap'](root, 'train', 0.5, read_meta=False, lens_distortion=True)
    c = d.camera
    assert c.model == model
    fx, fy, cx, cy, dist = want
    assert (c.fx, c.fy, c.cx, c.cy) == (fx / 2, fy / 2, cx / 2, cy / 2)   # scaled; the distortion terms are not
    assert c.dist == dist
    assert np.array_equal(d.K.numpy(), np.float32([[fx / 2, 0, cx / 2], [0, fy / 2, cy / 2], [0, 0, 1]]))
    assert d.img_wh == (20, 15)


@pytest.mark.parametrize('model', ['OPENCV_FISHEYE', 'FULL_OPENCV', 'FOV', 'RADIAL_FISHEYE'])
def test_colmap_refuses_other_models(tmp_path, model):
    from datasets import dataset_dict
    n = {'OPENCV_FISHEYE': 8, 'FULL_OPENCV': 12, 'FOV': 5, 'RADIAL_FISHEYE': 5}[model]
    root = _colmap(tmp_path, model, [30.0] * n)
    with pytest.raises(ValueError, match=model):
        dataset_dict['colmap'](root, 'train', 1.0, read_meta=False, lens_distortion=True)


def test_colmap_without_the_flag_is_unchanged(tmp_path):
    from datasets import dataset_dict
    from datasets.ray_utils import get_ray_directions
    root = _colmap(tmp_path, 'SIMPLE_RADIAL', [30.0, 20.0, 15.0, -0.1])
    d = dataset_dict['colmap'](root, 'train', 1.0, read_meta=False)
    assert d.camera is None
    assert torch.equal(d.directions, get_ray_directions(30, 40, d.K))
    # the distortion-free table of the flag is the same pinhole table until to(device) unprojects
    e = dataset_dict['colmap'](root, 'train', 1.0, read_meta=False, lens_distortion=True)
    assert torch.equal(e.K, d.K) and torch.equal(e.directions, d.directions)
    # without the flag the models it adds stay refused, as before
    root2 = _colmap(tmp_path / 'r', 'RADIAL', [30.0, 20.0, 15.0, -0.1, 0.0])
    with pytest.raises(ValueError, match="RADIAL"):
        dataset_dict['colmap'](root2, 'train', 1.0, read_meta=False)


def _ngp(tmp_path, **extra):
    meta = {'w': 40, 'h': 30, 'fl_x': 30.0, 'fl_y': 31.0, 'frames': [], **extra}
    tmp_path.mkdir(parents=True, exist_ok=True)
    with open(tmp_path / 'transforms.json', 'w') as f:
        json.dump(meta, f)
    return str(tmp_path)


def test_ngp_camera(tmp_path):
    from datasets import dataset_dict
    d = dataset_dict['ngp'](_ngp(tmp_path / 'a', cx=19.0, cy=14.5, k1=-0.2, k2=0.05, p1=0.001, p2=-0.002), 'train',
                            0.5, read_meta=False, lens_distortion=True)
    c = d.camera
    assert c.model == 'OPENCV' and (c.fx, c.fy, c.cx, c.cy) == (15.0, 15.5, 9.5, 7.25)
    assert c.dist == (-0.2, 0.05, 0.001, -0.002)
    assert np.array_equal(d.K.numpy(), np.float32([[15, 0, 9.5], [0, 15.5, 7.25], [0, 0, 1]]))
    # without cx cy k*: the centre and no distortion, the K of the flag-less loader
    e = dataset_dict['ngp'](_ngp(tmp_path / 'b'), 'train', 0.5, read_meta=False, lens_distortion=True)
    assert (e.camera.cx, e.camera.cy) == (10.0, 7.5) and not e.camera.has_distortion
    f = dataset_dict['ngp'](_ngp(tmp_path / 'b'), 'train', 0.5, read_meta=False)
    assert f.camera is None and torch.equal(e.K, f.K) and torch.equal(e.directions, f.directions)


def test_ngp_without_the_flag_is_unchanged(tmp_path):
    from datasets import dataset_dict
    from datasets.ray_utils import get_ray_directions
    d = dataset_dict['ngp'](_ngp(tmp_path, cx=3.0, cy=4.0, k1=-0.2, is_fisheye=True, k3=0.1), 'train', 1.0,
                            read_meta=False)
    assert d.camera is None
    assert np.array_equal(d.K.numpy(), np.float32([[30, 0, 20], [0, 31, 15], [0, 0, 1]]))
    assert torch.equal(d.directions, get_ray_directions(30, 40, d.K))


@pytest.mark.parametrize('extra, what', [({'is_fisheye': True}, 'is_fisheye'), ({'k3': 0.1}, 'k3'),
                                         ({'k4': -0.1}, 'k4')])
def test_ngp_refusals(tmp_path, extra, what):
    from datasets import dataset_dict
    with pytest.raises(ValueError, match=what):
        dataset_dict['ngp'](_ngp(tmp_path, **extra), 'train', 1.0, read_meta=False, lens_distortion=True)


def test_camera_validation():
    from taichi_nerfs_b200.intrinsics import Camera
    with pytest.raises(ValueError, match="not supported"):
        Camera('FULL_OPENCV', 1.0, 1.0, 0.0, 0.0)
    with pytest.raises(ValueError, match="SIMPLE_RADIAL"):
        Camera('SIMPLE_RADIAL', 1.0, 1.0, 0.0, 0.0, (0.1, 0.2, 0.0, 0.0))
    with pytest.raises(ValueError, match="finite"):
        Camera('PINHOLE', 0.0, 1.0, 0.0, 0.0)


# ---- the reference --------------------------------------------------------------------------------------------------
CAMERAS = [((-0.25, 0.0, 0.0, 0.0), 800, 600, 700.0), ((-0.25, 0.06, 0.0, 0.0), 800, 600, 700.0),
           ((-0.2, 0.03, 0.002, -0.003), 800, 600, 650.0), ((0.1, 0.02, -0.001, 0.002), 400, 300, 380.0)]


@pytest.mark.parametrize("dist, W, H, f", CAMERAS)
def test_reference_inverse(dist, W, H, f):
    pix = torch.arange(W * H)
    xd, yd = ref.pixel_xd(pix, W, H, f, f * 1.01, W / 2 - 3.0, H / 2 + 2.0)
    xu, yu = ref.undistort(dist, xd, yd)
    x2, y2 = ref.distort(dist, xu, yu)
    assert float((x2 - xd).abs().max()) <= 1e-12 and float((y2 - yd).abs().max()) <= 1e-12
    a, b, c, d = ref.jacobian(dist, xu, yu)
    assert float((a * d - b * c).min()) > 0     # every pixel lies inside the fold


@pytest.mark.parametrize("dist", [c[0] for c in CAMERAS])
def test_reference_jacobian_against_central_differences(dist):
    g = torch.Generator().manual_seed(3)
    x, y = (torch.rand(500, generator=g, dtype=torch.float64) - 0.5) * 1.2, \
        (torch.rand(500, generator=g, dtype=torch.float64) - 0.5) * 0.9
    h = 1e-6
    J = ref.jacobian(dist, x, y)
    num = [(ref.distort(dist, x + h, y)[0] - ref.distort(dist, x - h, y)[0]) / (2 * h),
           (ref.distort(dist, x, y + h)[0] - ref.distort(dist, x, y - h)[0]) / (2 * h),
           (ref.distort(dist, x + h, y)[1] - ref.distort(dist, x - h, y)[1]) / (2 * h),
           (ref.distort(dist, x, y + h)[1] - ref.distort(dist, x, y - h)[1]) / (2 * h)]
    for a, b in zip(J, num):
        assert float((a - b).abs().max()) < 1e-8


def test_package_distortion_matches_reference():
    from taichi_nerfs_b200.intrinsics import Camera, distort_np
    c = Camera('OPENCV', 1.0, 1.0, 0.0, 0.0, (-0.2, 0.03, 0.002, -0.003))
    x, y = np.linspace(-0.8, 0.8, 33), np.linspace(0.6, -0.6, 33)
    a, b = distort_np(c, x, y)
    ra, rb = ref.distort(c.dist, torch.from_numpy(x), torch.from_numpy(y))
    assert np.array_equal(a, ra.numpy()) and np.array_equal(b, rb.numpy())


# ---- C-ABI ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def _cam(*p):
    return (C.c_double * 8)(*(list(p) + [0.0] * (8 - len(p))))


def test_intrinsics_argument_validation_needs_no_gpu(lib):
    fake, odd = C.c_void_p(0x10000), C.c_void_p(0x10004)
    ok = _cam(30.0, 30.0, 20.0, 15.0, -0.1)
    un = lib.ngp_camera_unproject
    # camera: size, model, parameters
    assert un(fake, 8, 0, 30, 1, ok, None, fake, None, None, None, None) < 0
    assert b"W and H" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 4, ok, None, fake, None, None, None, None) < 0
    assert b"camera model" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 0, ok, None, fake, None, None, None, None) < 0    # PINHOLE with a k1
    assert b"distortion term" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 1, _cam(0.0, 30.0, 20.0, 15.0), None, fake, None, None, None, None) < 0
    assert b"focal" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 1, _cam(float('nan'), 30.0, 20.0, 15.0), None, fake, None, None, None, None) < 0
    assert b"finite" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 1, None, None, fake, None, None, None, None) < 0
    # counts, pointers, alignment
    assert un(fake, -1, 40, 30, 1, ok, None, fake, None, None, None, None) < 0
    assert un(None, 8, 40, 30, 1, ok, None, fake, None, None, None, None) < 0
    assert b"W * H" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 1, ok, None, None, None, None, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 1, ok, odd, fake, None, None, None, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert un(fake, 8, 40, 30, 1, ok, None, fake, odd, None, None, None) < 0
    assert un(None, 0, 40, 30, 1, ok, None, None, None, None, None, None) < 0   # n must be W * H without indices
    assert un(fake, 0, 40, 30, 1, ok, None, None, None, None, None, None) == 0
    # counts whose launch grid would not fit: refused, not truncated
    assert un(fake, 2 ** 31, 40, 30, 1, ok, None, fake, None, None, None, None) < 0
    assert b"2^31" in lib.ngp_last_error()
    big = _cam(30.0, 30.0, 20.0, 15.0, -0.1)
    assert un(None, 2 ** 24 * 2 ** 24, 2 ** 24, 2 ** 24, 1, big, None, fake, None, None, None, None) < 0
    assert b"2^31" in lib.ngp_last_error()
    # gradient
    gr = lib.ngp_intrinsics_grad
    args = [fake, fake, fake, 8, None, 64, fake, fake, fake, None, 4, fake, 40, 30, 1, ok, fake, fake, 8, None, None]

    def g(**kw):
        a = list(args)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return gr(*a)
    assert g(a3=-1) < 0 and g(a5=-1) < 0 and g(a18=-1) < 0
    assert g(a10=0) < 0
    assert b"n_img" in lib.ngp_last_error()
    assert g(a6=None) < 0 and g(a16=None) < 0 and g(a17=None) < 0
    assert b"null" in lib.ngp_last_error()
    assert g(a0=None) < 0
    assert g(a17=odd) < 0 and g(a9=odd) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert g(a14=7) < 0
    assert g(a3=2 ** 31) < 0 and g(a18=2 ** 31) < 0
    assert b"2^31" in lib.ngp_last_error()
    assert g(a3=0, a0=None, a1=None, a2=None) == 0
    # Adam
    ad = lib.ngp_intrinsics_adam
    assert ad(fake, fake, -1, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, None, None) < 0
    assert ad(fake, fake, 2 ** 31, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, None, None) < 0
    assert b"2^31" in lib.ngp_last_error()
    assert ad(fake, fake, 8, fake, fake, None, None, 0.1, 0.9, 0.999, 1e-15, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert ad(fake, None, 8, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, None, None) < 0
    assert ad(odd, fake, 8, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, None, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert ad(fake, fake, 8, fake, fake, None, fake, float('inf'), 0.9, 0.999, 1e-15, None, None) < 0
    assert b"lr_ratio" in lib.ngp_last_error()


def test_new_kernels_compile_without_spills():
    """ptxas for sm_90a: no spill stores or loads in the three kernels of csrc/camera.cu."""
    import subprocess
    from taichi_nerfs_b200 import build
    src = os.path.join(build.CSRC, 'camera.cu')
    out = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, '-Xptxas', '-v', '-c', src, '-o', os.devnull],
                         capture_output=True, text=True, check=True).stderr
    kernels = out.split("Compiling entry function")[1:]
    assert len(kernels) == 3
    for k in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in k, k
