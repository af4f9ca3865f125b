"""train.py on datasets read from disk: views of the reference's shipped trained Lego model (the teacher) exported in
the Blender layout and in the COLMAP layout, then trained through ``--dataset_name nerf`` / ``colmap``."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _teacher():
    import __graft_entry__ as g
    if not g.stage_lego_fixture():
        pytest.skip("shipped Lego weights could not be staged")
    from datasets.teacher import load_teacher
    return load_teacher(torch.device('cuda'))


@torch.no_grad()
def _render(teacher, ds):
    """[n, H*W, 3] colours on white and [n, H*W] opacities of the teacher at the dataset's poses."""
    from datasets.ray_utils import get_rays
    from modules.rendering import render
    rgbs, ops = [], []
    for pose in ds.poses:
        o, d = get_rays(ds.directions, pose)
        with torch.autocast('cuda', dtype=torch.float16):
            res = render(teacher, o, d, test_time=True, T_threshold=1e-2, exp_step_factor=0.0)
        rgbs.append(res['rgb'].float().clamp(0, 1))
        ops.append(res['opacity'].float().clamp(0, 1))
    return torch.stack(rgbs), torch.stack(ops)


def _u8(x):
    return (x.clamp(0, 1) * 255 + 0.5).to(torch.uint8).cpu().numpy()


def _export_blender(root, teacher, n_train, n_test, downsample):
    """Blender layout at radius 1.5 (NeRFDataset rescales every camera to 1.5): RGBA PNGs whose alpha is the teacher's
    opacity and whose colour is the un-premultiplied teacher colour, so that blending onto white gives the render."""
    from datasets.teacher import TeacherLego
    from PIL import Image
    focal = 1111.111
    for split, n in (('train', n_train), ('test', n_test)):
        ds = TeacherLego(n_images=n, radius=1.5, split=split, downsample=downsample).to('cuda')
        rgb, a = _render(teacher, ds)
        w, h = ds.img_wh
        straight = torch.where(a[..., None] > 1e-4, (rgb - (1 - a[..., None])) / a[..., None].clamp_min(1e-4), 0.)
        os.makedirs(os.path.join(root, split), exist_ok=True)
        frames = []
        for i in range(n):
            rgba = np.concatenate([_u8(straight[i]), _u8(a[i])[:, None]], 1).reshape(h, w, 4)
            Image.fromarray(rgba).save(os.path.join(root, split, f'r_{i}.png'))
            c2w = ds.poses[i].cpu().double().numpy().copy()
            c2w[:, 1:3] *= -1                                   # [right down front] -> [right up back]
            frames.append({'file_path': f'./{split}/r_{i}',
                           'transform_matrix': np.concatenate([c2w, [[0, 0, 0, 1]]], 0).tolist()})
        with open(os.path.join(root, f'transforms_{split}.json'), 'w') as f:
            json.dump({'camera_angle_x': 2 * math.atan(400 / focal), 'frames': frames}, f)


def test_blender_layout_trains_like_teacher_protocol(tmp_path, monkeypatch, capsys):
    """--dataset_name nerf --graph_step on exported teacher views: held-out PSNR within 0.5 dB of
    psnr.train_vs_teacher at the same step count, views, resolution and batch."""
    import train
    from taichi_nerfs_b200.psnr import train_vs_teacher
    teacher = _teacher()
    steps, n_train, n_test, down = 1500, 32, 2, 0.25
    root = str(tmp_path / 'lego_blender')
    _export_blender(root, teacher, n_train, n_test, down)
    monkeypatch.chdir(tmp_path)
    psnrs = train.main(['--dataset_name', 'nerf', '--root_dir', root, '--downsample', str(down), '--half_opt',
                        '--graph_step', '--max_steps', str(steps - 1)])
    disk = sum(psnrs) / len(psnrs)
    r = train_vs_teacher(torch.device('cuda'), steps=steps, train_views=n_train, test_views=n_test, downsample=down,
                         teacher=teacher)
    with capsys.disabled():
        print(f"\nblender layout: train.py --dataset_name nerf --graph_step {disk:.2f} dB {psnrs}; "
              f"train_vs_teacher {r['psnr']:.2f} dB {r['psnr_views']}")
    assert len(psnrs) == n_test
    assert disk >= r['psnr'] - 0.5


def _export_colmap(root, teacher, n_views, wh):
    """COLMAP layout (PINHOLE camera, images/, sparse/0/*.bin) of teacher views composited onto black, with a sparse
    point cloud inside the Lego box (ColmapDataset centres the poses on its mean)."""
    from colmap_writer import rotmat2qvec, write_model
    from datasets.teacher import TeacherLego
    from PIL import Image
    focal = 1111.111 * wh / 800
    ds = TeacherLego(n_images=n_views, radius=1.396, split='train', img_wh=(wh, wh), focal=focal).to('cuda')
    rgb, a = _render(teacher, ds)
    premult = rgb - (1 - a[..., None])                        # the same render over black
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    imgs = []
    for i in range(n_views):
        name = f'view_{i:03d}.png'
        Image.fromarray(_u8(premult[i]).reshape(wh, wh, 3)).save(os.path.join(root, 'images', name))
        c2w = ds.poses[i].cpu().double().numpy()
        R = c2w[:, :3].T
        imgs.append((i + 1, rotmat2qvec(R), -R @ c2w[:, 3], 1, name, np.zeros((0, 2)), np.zeros(0, np.int64)))
    pts = np.random.default_rng(0).uniform(-0.3, 0.3, (200, 3))
    write_model(os.path.join(root, 'sparse', '0'), [(1, 'PINHOLE', wh, wh, [focal, focal, wh / 2, wh / 2])], imgs,
                [(k + 1, p, [128, 128, 128], 0.5, [1], [0]) for k, p in enumerate(pts)])


def test_colmap_layout_trains_at_real_scene_settings(tmp_path, monkeypatch, capsys):
    """--dataset_name colmap --scale 16 (several cascades, exp_step_factor 1/256, black background): the loss falls
    over a few hundred steps and the evaluation line is printed."""
    import train
    from taichi_nerfs_b200.trainer import NGPTrainer
    teacher = _teacher()
    root = str(tmp_path / 'scene')
    _export_colmap(root, teacher, 24, 128)
    losses = []

    class Recording(NGPTrainer):
        def step(self, *a, **k):
            loss, res = super().step(*a, **k)
            losses.append(float(loss.detach()))
            return loss, res

    monkeypatch.setattr(train, 'NGPTrainer', Recording)
    monkeypatch.chdir(tmp_path)
    psnrs = train.main(['--dataset_name', 'colmap', '--root_dir', root, '--scale', '16', '--half_opt',
                        '--batch_size', '4096', '--max_steps', '400'])
    out = capsys.readouterr().out
    with capsys.disabled():
        print(f"\ncolmap layout, scale 16: loss {np.mean(losses[:20]):.5f} (first 20 steps) -> "
              f"{np.mean(losses[-20:]):.5f} (last 20); held-out PSNR {psnrs}")
    assert 'evaluation: psnr_avg=' in out
    assert len(psnrs) == 3 and all(math.isfinite(p) for p in psnrs)          # views 0, 8, 16 of 24
    assert np.mean(losses[-50:]) < 0.5 * np.mean(losses[:20])
