"""Known-answer test: render the reference's SHIPPED, TRAINED Lego deployment model through the oracle.

The only real fixture the reference ships is its mobile-demo model
(deployment/InstantNGP/taichi_ngp/compiled/*.bin: hash grid L=4 F=4 32->128 T=2^21, 16-wide MLPs,
occupancy bitfield, pose, pixel directions).  Rendering it end to end with the oracle's
ray/AABB -> march -> dense hash indexing -> SH -> MLP weight layout -> compositing
(restating deployment/InstantNGP/taichi_ngp/kernels.py:262-571 and new_kernels.py:4-18) must produce
the yellow Lego bulldozer; any indexing / layout mistake produces noise.  This pins the oracle against
the reference's own artefact (test infrastructure).  The model is stored shrunk under tests/golden/
(lego_deployment.npz + lego_table_level3.npz, made by tests/golden/make_golden.py: the hash-table entries a render
through the occupancy grid can read, in fp16); stage() rebuilds the six .bin files from it under oracle/_ref/.

    NGP_REFERENCE=<taichi-nerfs checkout> python -m oracle.kat_lego
        # writes tests/golden/lego_kat.png + lego_kat_stats.json from the reference's ORIGINAL .bin files; it refuses
        # to run without them, so the golden image is never re-derived from the shrunk copy
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF_DIR = os.path.join(ROOT, "oracle", "_ref", "lego_deployment")   # git-ignored, rebuilt by stage()
FILES = ("hash_embedding", "sigma_weights", "rgb_weights", "density_bitfield", "pose", "directions")
TABLE_ENTRIES, TABLE_FEATURES = 2794024, 4     # make_hash_layout(2 ** 21, 4, 32, 128, 4)


def _write_bin(path, code, a):
    """[int32 dtype code][int32 numel][payload]; written to a temporary name first so a reader never sees half."""
    tmp = f"{path}.{os.getpid()}.tmp"
    with open(tmp, "wb") as f:
        f.write(np.array([code, a.size], np.int32).tobytes())
        f.write(np.ascontiguousarray(a).tobytes())
    os.replace(tmp, path)


def stage(dest=REF_DIR):
    """Rebuild the six deployment .bin files of the shipped Lego model in `dest` from the golden data (once);
    hash-table entries outside the stored set are zero.  Returns `dest`."""
    if all(os.path.exists(os.path.join(dest, n + ".bin")) for n in FILES):
        return dest
    os.makedirs(dest, exist_ok=True)
    g = np.load(os.path.join(GOLDEN, "lego_deployment.npz"))
    fine = np.load(os.path.join(GOLDEN, "lego_table_level3.npz"))["table_fine"]
    mask = np.unpackbits(g["table_mask"])[:TABLE_ENTRIES].astype(bool)
    table = np.zeros((TABLE_ENTRIES, TABLE_FEATURES), np.float32)
    table[mask] = np.concatenate([g["table_coarse"], fine]).astype(np.float32)   # entries in index order
    dx, dy = g["dir_x"], g["dir_y"]
    dirs = np.stack(np.broadcast_arrays(dx[None, :], dy[:, None], np.float32(1)), -1).astype(np.float32)
    bits = np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"]
    _write_bin(os.path.join(dest, "hash_embedding.bin"), 0, table.reshape(-1))
    _write_bin(os.path.join(dest, "sigma_weights.bin"), 0, g["sigma_weights"].astype(np.float32))
    _write_bin(os.path.join(dest, "rgb_weights.bin"), 0, g["rgb_weights"].astype(np.float32))
    _write_bin(os.path.join(dest, "density_bitfield.bin"), 4, bits.view(np.uint32))
    _write_bin(os.path.join(dest, "pose.bin"), 0, g["pose"].astype(np.float32))
    _write_bin(os.path.join(dest, "directions.bin"), 0, dirs.reshape(-1))
    return dest


def read_bin(path):
    """[int32 dtype][int32 numel][payload]  (taichi_ngp.py:34-65, utils.cpp:100-120)."""
    raw = np.fromfile(path, dtype=np.uint8)
    code, numel = raw[:8].view(np.int32)
    dt = {0: np.float32, 1: np.float16, 2: np.int32, 3: np.int16, 4: np.uint32, 5: np.uint16}[int(code)]
    return raw[8:].view(dt)[:numel]


def sh16(d):
    sys.path.insert(0, ROOT)
    from oracle import oracle as O
    return O.dir_encode(d)


def deployment_mlp(emb, dirs, sigma_w, rgb_w):
    """sigma_rgb_layer, kernels.py:449-518: sigma net 16->16(relu)->16, rgb net [SH16|h16]->16(relu)->3."""
    W1 = sigma_w[:256].reshape(16, 16)          # temp_i = sum_j emb_j * w[i*16+j]
    W2 = sigma_w[256:512].reshape(16, 16)       # out_j += relu(temp_i) * w[256 + j*16 + i]
    h = np.maximum(emb @ W1.T, 0) @ W2.T
    sigma = np.exp(h[:, 0])
    d = dirs / np.linalg.norm(dirs, axis=1, keepdims=True)
    sh = sh16(((d + 1) / 2).astype(np.float32))  # dir_encode_func, kernels.py:139-172
    x = np.concatenate([sh, h], 1).astype(np.float32)
    W3 = rgb_w[:512].reshape(16, 32)
    W4 = rgb_w[512:512 + 48].reshape(3, 16)     # s_c += relu(temp_i) * w[512 + c*16 + i]
    o = np.maximum(x @ W3.T, 0) @ W4.T
    return sigma.astype(np.float32), (1 / (1 + np.exp(-o))).astype(np.float32)


def render(step=2, T_threshold=1e-2, max_samples=1024, src=None):
    """Render the shipped view from the six .bin files in `src` (default: the copy stage() rebuilds)."""
    sys.path.insert(0, ROOT)
    src = src or stage()
    from oracle import oracle as O
    from taichi_nerfs_b200.layout import make_hash_layout
    emb_table = read_bin(os.path.join(src, "hash_embedding.bin"))
    sigma_w = read_bin(os.path.join(src, "sigma_weights.bin"))
    rgb_w = read_bin(os.path.join(src, "rgb_weights.bin"))
    bits = read_bin(os.path.join(src, "density_bitfield.bin")).view(np.uint8)
    pose = read_bin(os.path.join(src, "pose.bin")).reshape(3, 4)
    directions = read_bin(os.path.join(src, "directions.bin")).reshape(600, 300, 3)  # (h, w) row-major
    lay = make_hash_layout(2 ** 21, 4, 32, 128, 4)
    assert lay.total_param_size == emb_table.size

    dirs_cam = directions[::step, ::step].reshape(-1, 3)
    h, w = directions[::step, ::step].shape[:2]
    rays_d = (dirs_cam @ pose[:, :3].T).astype(np.float32)        # new_kernels.py:12
    rays_o = np.tile(pose[:, 3], (rays_d.shape[0], 1)).astype(np.float32)
    hits = O.ray_aabb_intersect(rays_o, rays_d, 0.5)
    noise = np.zeros(rays_d.shape[0], np.float32)
    rays_a, xyzs, sdirs, deltas, ts, S = O.raymarching_train(rays_o, rays_d, hits, bits, noise, 1, 0.5, 0.0, 128,
                                                             max_samples)
    emb = O.hash_encode_fwd((xyzs + 0.5).astype(np.float32), emb_table, lay)  # kernels.py:397 (xyz + 0.5)
    sigma, rgbs = deployment_mlp(emb, sdirs, sigma_w, rgb_w)
    tot, opacity, depth, rgb, ws = O.composite_train_fwd(sigma, rgbs, deltas, ts, rays_a, T_threshold)
    return rgb.reshape(h, w, 3), opacity.reshape(h, w), S / rays_d.shape[0], rays_a[:, 2].reshape(h, w)


def stats(rgb, opacity, spr):
    obj = opacity > 0.5
    col = rgb[obj].mean(0) / np.maximum(opacity[obj].mean(), 1e-6)
    return {"coverage": float(obj.mean()), "semi_transparent_fraction": float(((opacity > 0.05) & (opacity < 0.95)).mean()),
            "object_mean_rgb": [float(c) for c in col], "samples_per_ray": float(spr),
            "opacity_max": float(opacity.max())}


def main():
    src = os.path.join(os.environ.get("NGP_REFERENCE", ""), "deployment", "InstantNGP", "taichi_ngp", "compiled")
    if not os.environ.get("NGP_REFERENCE") or not all(os.path.exists(os.path.join(src, n + ".bin")) for n in FILES):
        sys.exit("set NGP_REFERENCE to a taichi-nerfs checkout: the golden image is made from the original model files")
    rgb, opacity, spr, _ = render(src=src)
    st = stats(rgb, opacity, spr)
    out = os.path.join(ROOT, "tests", "golden")
    from PIL import Image
    Image.fromarray((np.clip(rgb + (1 - opacity)[..., None], 0, 1) * 255).astype(np.uint8)).save(
        os.path.join(out, "lego_kat.png"))
    with open(os.path.join(out, "lego_kat_stats.json"), "w") as f:
        json.dump(st, f, indent=1)
    print(st)


if __name__ == "__main__":
    main()
