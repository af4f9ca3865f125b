"""Tiny on-disk datasets for the disk loaders' tests, and the reference loaders' outputs on them.

    python tests/golden/make_dataset_golden.py fixtures                       # writes tests/golden/datasets/
    python tests/golden/make_dataset_golden.py golden <taichi-nerfs checkout> # writes tests/golden/datasets_golden.npz

Both outputs are committed, the image files included, so that PNG and JPEG decoding is pinned by the files and not by
the encoder that wrote them; no test runs this script.  ``golden`` imports the reference's ``datasets`` package from
the checkout with two shims for packages it needs that are not installed here: ``imageio.imread`` (PIL decoding to a
uint8 array, which is what imageio's PIL plugin does for PNG and JPEG) and kornia's ``create_meshgrid`` (unnormalised
pixel coordinates, x then y, from ``torch.linspace``).  It stores, per (format, split), the reference's ``K``,
``img_wh``, ``directions``, ``poses`` and ``rays`` and, for images with an alpha channel, the alpha resized as the
loaders here resize it.

Fixtures (one per format and per name-dependent branch):
  nerf_blender/            Blender layout, 32x32 RGBA PNGs; train 3 / val 1 / test 2; read at downsample 0.02 (16x16)
  Synthetic_NeRF/Lego/     NSVF layout (Synthetic intrinsics, bbox.txt, the Lego x1.1 bound), 32x32 RGBA PNGs,
                           0_/1_/2_ prefixes and test_traj.txt; read at downsample 0.02
  ngp_scene/               instant-ngp transforms.json, 40x30 RGB PNGs, one frame without its file; downsample 0.5
  360_v2/garden/           COLMAP binary model (PINHOLE 64x48), ten JPEGs in images_4/ (16x12), names not in id
                           order; read at downsample 0.25
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, 'datasets')
GOLDEN = os.path.join(HERE, 'datasets_golden.npz')

# (loader name, directory under tests/golden/datasets, split, downsample)
CASES = ([('nerf', 'nerf_blender', s, 0.02) for s in ('train', 'val', 'test', 'trainval')]
         + [('nsvf', 'Synthetic_NeRF/Lego', s, 0.02)
            for s in ('train', 'val', 'test', 'trainval', 'trainvaltest', 'test_traj')]
         + [('ngp', 'ngp_scene', 'train', 0.5)]
         + [('colmap', '360_v2/garden', s, 0.25) for s in ('train', 'test', 'test_traj')])


def case_key(name, root, split):
    return f"{name}__{root.replace('/', '_')}__{split}"


def smooth_image(h, w, seed, alpha):
    """uint8 [h, w, 3|4]: low-frequency colour ramps and a soft disc of alpha (so PNGs stay small)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w] / np.array([h, w])[:, None, None]
    c = rng.uniform(0.2, 0.8, (3, 3))
    rgb = np.stack([c[i, 0] + 0.2 * np.sin(2 * np.pi * (c[i, 1] * x + c[i, 2] * y)) for i in range(3)], -1)
    out = [np.clip(rgb * 255 + 0.5, 0, 255)]
    if alpha:
        r = np.hypot(x - 0.5 - 0.1 * c[0, 0], y - 0.5)
        out.append(np.clip((0.35 - r) * 6, 0, 1)[..., None] * 255 + 0.5)
    return np.concatenate(out, -1).astype(np.uint8)


def look_at(pos, target=(0, 0, 0), up=(0, 0, 1)):
    """3x4 camera-to-world [right, down, front, position] (OpenCV axes) looking from ``pos`` at ``target``."""
    pos = np.asarray(pos, float)
    front = np.asarray(target, float) - pos
    front /= np.linalg.norm(front)
    right = np.cross(front, up)
    right /= np.linalg.norm(right)
    down = np.cross(front, right)
    return np.stack([right, down, front, pos], 1)


def ring(n, radius, height, phase=0.3):
    return [(radius * np.cos(phase + 2 * np.pi * i / n), radius * np.sin(phase + 2 * np.pi * i / n),
             height + 0.1 * np.sin(i)) for i in range(n)]


def save_png(path, arr):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(arr).save(path, optimize=True)


def write_fixtures():
    from PIL import Image
    sys.path.insert(0, os.path.dirname(HERE))
    from colmap_writer import rotmat2qvec, write_model

    # Blender: c2w columns [right, up, back]
    root = os.path.join(DATA, 'nerf_blender')
    seed = 0
    for split, n in (('train', 3), ('val', 1), ('test', 2)):
        frames = []
        for i, p in enumerate(ring(n, 3.6, 1.9, phase=0.3 + len(split))):
            c2w = look_at(p)
            c2w[:, 1:3] *= -1
            m = np.concatenate([c2w, [[0, 0, 0, 1]]], 0)
            frames.append({'file_path': f'./{split}/r_{i}', 'rotation': 0.0, 'transform_matrix': m.tolist()})
            save_png(os.path.join(root, split, f'r_{i}.png'), smooth_image(32, 32, seed, True))
            seed += 1
        with open(os.path.join(root, f'transforms_{split}.json'), 'w') as f:
            json.dump({'camera_angle_x': 0.6911112070083618, 'frames': frames}, f, indent=1)

    # NSVF Synthetic: OpenCV c2w in scene units, bbox + intrinsics
    root = os.path.join(DATA, 'Synthetic_NeRF', 'Lego')
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, 'bbox.txt'), 'w') as f:
        f.write('-0.637787 -1.140016 -0.344656 0.633744 1.148737 1.002206 0.010000\n')
    with open(os.path.join(root, 'intrinsics.txt'), 'w') as f:
        f.write('1111.111 400.0 400.0 0.\n0. 0. 0.\n0.\n1.\n800 800\n')
    for prefix, n in (('0', 3), ('1', 1), ('2', 2)):
        for i, p in enumerate(ring(n, 3.2, 1.5, phase=int(prefix) + 0.7)):
            m = np.concatenate([look_at(p), [[0, 0, 0, 1]]], 0)
            os.makedirs(os.path.join(root, 'pose'), exist_ok=True)
            np.savetxt(os.path.join(root, 'pose', f'{prefix}_{i:04d}.txt'), m)
            save_png(os.path.join(root, 'rgb', f'{prefix}_{i:04d}.png'), smooth_image(32, 32, seed, True))
            seed += 1
    traj = np.stack([np.concatenate([look_at(p), [[0, 0, 0, 1]]], 0) for p in ring(4, 3.0, 1.0)])
    np.savetxt(os.path.join(root, 'test_traj.txt'), traj.reshape(len(traj), 16))

    # instant-ngp: one transforms.json, RGB images, a frame without its file
    root = os.path.join(DATA, 'ngp_scene')
    frames = []
    for i, p in enumerate(ring(4, 2.5, 0.8)):
        c2w = look_at(p)
        c2w[:, 1:3] *= -1
        frames.append({'file_path': f'images/{i:03d}.png',
                       'transform_matrix': np.concatenate([c2w, [[0, 0, 0, 1]]], 0).tolist()})
        if i != 2:
            save_png(os.path.join(root, 'images', f'{i:03d}.png'), smooth_image(30, 40, seed, False))
        seed += 1
    with open(os.path.join(root, 'transforms.json'), 'w') as f:
        json.dump({'w': 40, 'h': 30, 'fl_x': 35.5, 'fl_y': 36.25, 'frames': frames}, f, indent=1)

    # COLMAP 360_v2: PINHOLE camera, images named out of id order, JPEGs in images_4/
    root = os.path.join(DATA, '360_v2', 'garden')
    rng = np.random.default_rng(5)
    names = [f'DSC{k:05d}.JPG' for k in rng.permutation(10) + 7000]
    imgs = []
    for i, (name, p) in enumerate(zip(names, ring(10, 4.0, 1.2))):
        c2w = look_at(p, target=(0.2, -0.1, 0.3))
        R = c2w[:, :3].T
        t = -R @ c2w[:, 3]
        imgs.append((i + 1, rotmat2qvec(R), t, 1, name, rng.uniform(0, 64, (3, 2)), [1, 2, -1]))
        img = Image.fromarray(smooth_image(12, 16, seed, False))
        os.makedirs(os.path.join(root, 'images_4'), exist_ok=True)
        img.save(os.path.join(root, 'images_4', name), quality=90)
        seed += 1
    pts = [(k + 1, rng.normal(0, 0.5, 3), rng.integers(0, 255, 3), 0.5, [1, 2], [0, 1]) for k in range(40)]
    write_model(os.path.join(root, 'sparse', '0'), [(1, 'PINHOLE', 64, 48, [52.25, 51.75, 32.5, 23.75])], imgs, pts)


def import_reference(ref):
    """The reference's ``datasets`` package, with the imageio and kornia shims described above."""
    import torch
    from PIL import Image

    imageio = types.ModuleType('imageio')
    imageio.imread = lambda p: np.asarray(Image.open(p))
    kornia = types.ModuleType('kornia')

    def create_meshgrid(h, w, normalized_coordinates=True, device='cpu'):
        assert not normalized_coordinates
        xs = torch.linspace(0, w - 1, w, device=device)
        ys = torch.linspace(0, h - 1, h, device=device)
        return torch.stack(torch.meshgrid([xs, ys], indexing='ij'), -1).permute(1, 0, 2)[None]

    kornia.create_meshgrid = create_meshgrid
    sys.modules['imageio'] = imageio
    sys.modules['kornia'] = kornia
    for k in [k for k in sys.modules if k == 'datasets' or k.startswith('datasets.')]:
        del sys.modules[k]
    sys.path.insert(0, os.path.abspath(ref))
    import datasets
    assert os.path.abspath(datasets.__file__).startswith(os.path.abspath(ref))
    return datasets


def write_golden(ref):
    import cv2
    from PIL import Image
    ds = import_reference(ref)
    out = {}
    for name, root, split, down in CASES:
        d = ds.dataset_dict[name](root_dir=os.path.join(DATA, root), split=split, downsample=down)
        key = case_key(name, root, split)
        out[key + '__K'] = d.K.numpy()
        out[key + '__img_wh'] = np.array(d.img_wh)
        out[key + '__directions'] = d.directions.numpy()
        out[key + '__poses'] = d.poses.numpy()
        rays = d.rays.numpy() if hasattr(d.rays, 'numpy') else np.zeros((0,), np.float32)
        out[key + '__rays'] = rays
        print(key, d.K.numpy().ravel()[[0, 2, 4, 5]], d.img_wh, tuple(d.poses.shape), rays.shape)
    # alpha of the RGBA fixtures, resized as datasets/color_utils.py resizes it (the reference drops it)
    for name, root, split, down in CASES:
        if name not in ('nerf', 'nsvf') or split == 'test_traj':
            continue
        d = ds.dataset_dict[name](root_dir=os.path.join(DATA, root), split=split, downsample=down)
        paths = alpha_paths(name, os.path.join(DATA, root), split)
        out[case_key(name, root, split) + '__alpha'] = np.stack([
            cv2.resize(np.ascontiguousarray(np.asarray(Image.open(p))[..., 3].astype(np.float32) / 255.0),
                       d.img_wh).reshape(-1) for p in paths])
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN, os.path.getsize(GOLDEN), 'bytes')


def alpha_paths(name, root, split):
    import glob
    if name == 'nsvf':
        pre = {'train': '0_', 'val': '1_', 'test': '2_', 'trainval': '[0-1]_', 'trainvaltest': '[0-2]_'}[split]
        return sorted(glob.glob(os.path.join(root, 'rgb', pre + '*.png')))
    frames = []
    for s in (('train', 'val') if split == 'trainval' else (split,)):
        with open(os.path.join(root, f'transforms_{s}.json')) as f:
            frames += json.load(f)['frames']
    return [os.path.join(root, fr['file_path'] + '.png') for fr in frames]


if __name__ == '__main__':
    if sys.argv[1:2] == ['fixtures']:
        write_fixtures()
    elif sys.argv[1:2] == ['golden'] and len(sys.argv) == 3:
        write_golden(sys.argv[2])
    else:
        sys.exit(__doc__)
