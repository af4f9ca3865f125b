"""Generates the small golden fixtures under tests/golden/ from the reference checkout.

Needs a reference checkout, named by the environment variable NGP_REFERENCE:
    NGP_REFERENCE=<taichi-nerfs checkout> python tests/golden/make_golden.py
Outputs (committed):
  lego_bitfield.npz      — the trained Lego occupancy bitfield shipped with the reference's mobile
                           demo (deployment/InstantNGP/taichi_ngp/compiled/density_bitfield.bin,
                           128^3 bits, 3.94 % occupied), zlib-compressed.  Used as the "occupancy (A)"
                           workload of BASELINE.md §4 and as a real-world marching fixture.
  layout_constants.json  — hash-layout constants printed by the reference itself
                           (notebooks/pipeline.ipynb cell 1; deployment/InstantNGP/utils/app_fp32.cpp:70-71).
  lego_deployment.npz,   — the reference's shipped trained Lego deployment model (compiled/*.bin), shrunk to what
  lego_table_level3.npz    a render can read: the MLP weights, pose and pixel-direction axes exactly; of the 44 MB
                           hash table only the entries at the grid corners of occupied cells (190,699 of 2,794,024),
                           rounded to fp16.  Samples exist only in occupied cells, so every render through the
                           occupancy grid reads only these entries.  oracle/kat_lego.py rebuilds the six .bin files
                           from them (the other entries zero).
"""
import json
import os
import sys

import numpy as np

REF = os.environ.get("NGP_REFERENCE", "")
HERE = os.path.dirname(os.path.abspath(__file__))


def read_bin(path):
    """[int32 dtype][int32 numel][payload] container (deployment/InstantNGP/taichi_ngp/taichi_ngp.py:34-65)."""
    raw = np.fromfile(path, dtype=np.uint8)
    dtype_code, numel = raw[:8].view(np.int32)
    np_dtype = {0: np.float32, 1: np.float16, 2: np.int32, 3: np.int16, 4: np.uint32, 5: np.uint16}[int(dtype_code)]
    return raw[8:].view(np_dtype)[:numel]


def reachable_entries(bits, lay):
    """Mask over the hash-table entries that a sample inside an occupied cell of the 128^3 bitfield can touch: the
    8 corners of its grid cell at every level (oracle/ngp_oracle.c hash_corners: p = x * scale + 0.5 on x = xyz + 0.5
    in [0, 1], dense index p0 + p1 R + p2 R^2 mod map size); the cell bounds are widened by 1e-5 for fp32 rounding."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import oracle as O
    occ = np.unpackbits(bits, bitorder="little")
    c = O.morton3d_invert(np.nonzero(occ)[0].astype(np.int32)).astype(np.int64)
    mask = np.zeros(lay.total_entries, bool)
    for lv in range(lay.levels):
        s, R, off, ms = lay.scales[lv], lay.resolutions[lv], lay.offsets[lv], lay.map_sizes[lv]
        lo = np.floor((c / 128 - 1e-5) * s + 0.5).astype(np.int64)
        hi = np.floor(((c + 1) / 128 + 1e-5) * s + 0.5).astype(np.int64) + 1
        for a in range(3):
            for b in range(3):
                for d in range(3):
                    g = np.stack([lo[:, 0] + a, lo[:, 1] + b, lo[:, 2] + d], 1)
                    g = g[(g <= hi).all(1)]
                    mask[off + (g[:, 0] + g[:, 1] * R + g[:, 2] * R * R) % ms] = True
    return mask


def lego_model(comp):
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from taichi_nerfs_b200.layout import make_hash_layout
    lay = make_hash_layout(2 ** 21, 4, 32, 128, 4)
    emb = read_bin(os.path.join(comp, "hash_embedding.bin")).reshape(-1, 4)
    bits = read_bin(os.path.join(comp, "density_bitfield.bin")).view(np.uint8)
    mask = reachable_entries(bits, lay)
    fine = np.arange(lay.total_entries) >= lay.offsets[3]
    d = read_bin(os.path.join(comp, "directions.bin")).reshape(600, 300, 3)
    dir_x, dir_y = d[0, :, 0].copy(), d[:, 0, 1].copy()
    # the directions are a separable pinhole grid (x per column, y per row, z = 1)
    assert (d[..., 0] == dir_x[None]).all() and (d[..., 1] == dir_y[:, None]).all() and (d[..., 2] == 1).all()
    np.savez_compressed(os.path.join(HERE, "lego_deployment.npz"),
                        sigma_weights=read_bin(os.path.join(comp, "sigma_weights.bin")),
                        rgb_weights=read_bin(os.path.join(comp, "rgb_weights.bin")),
                        pose=read_bin(os.path.join(comp, "pose.bin")), dir_x=dir_x, dir_y=dir_y,
                        table_mask=np.packbits(mask), table_coarse=emb[mask & ~fine].astype(np.float16))
    np.savez_compressed(os.path.join(HERE, "lego_table_level3.npz"), table_fine=emb[mask & fine].astype(np.float16))
    print("hash entries kept:", int(mask.sum()), "of", lay.total_entries)


def main():
    comp = os.path.join(REF, "deployment/InstantNGP/taichi_ngp/compiled")
    lego_model(comp)
    bits = read_bin(os.path.join(comp, "density_bitfield.bin")).view(np.uint8)
    assert bits.size == 128 ** 3 // 8
    np.savez_compressed(os.path.join(HERE, "lego_bitfield.npz"), bitfield=bits)
    pose = read_bin(os.path.join(comp, "pose.bin")).reshape(3, 4)

    # constants the reference prints / hard-codes
    consts = {
        "source": {
            "lego_16_1024": "notebooks/pipeline.ipynb cell 1 (per_level_scale, offset_, total_hash_size)",
            "deployment": "deployment/InstantNGP/utils/app_fp32.cpp:70-71, taichi_ngp/kernels.py (offsets)",
        },
        "lego_16_1024": {"per_level_scale": 1.3195079107728942, "total_entries": 5710032,
                         "total_params": 11420064},
        "deployment": {"total_params": 11176096, "offsets_entries": [0, 32768, 165424, 696872]},
        "deployment_pose": pose.tolist(),
        "bitfield_occupied_fraction": float(np.unpackbits(bits).mean()),
    }
    with open(os.path.join(HERE, "layout_constants.json"), "w") as f:
        json.dump(consts, f, indent=1)
    print("bitfield occupied:", consts["bitfield_occupied_fraction"])


if __name__ == "__main__":
    main()
