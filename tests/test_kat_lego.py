"""Known-answer test against the reference's shipped trained Lego deployment model (stored shrunk under tests/golden/,
rebuilt by oracle.kat_lego.stage())."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import kat_lego

def test_oracle_renders_the_shipped_lego_model():
    rgb, opacity, spr, counts = kat_lego.render(step=3)
    st = kat_lego.stats(rgb, opacity, spr)
    with open(os.path.join(GOLDEN, "lego_kat_stats.json")) as f:
        gold = json.load(f)
    # a trained scene is (almost) binary in opacity; wrong hash indexing / weight layout gives fog
    assert st["semi_transparent_fraction"] < 0.05
    assert abs(st["coverage"] - gold["coverage"]) < 0.03
    assert np.allclose(st["object_mean_rgb"], gold["object_mean_rgb"], atol=0.03)
    r, g, b = st["object_mean_rgb"]
    assert r > g > b and r - b > 0.3          # the yellow bulldozer on the tan base plate
    # opaque pixels can only occur where marching produced samples inside the trained occupancy grid
    assert not (opacity[counts == 0] > 1e-6).any()
    # image is not noise: neighbouring pixels agree (total variation far below that of random colours)
    tv = np.abs(np.diff(rgb, axis=0)).mean() + np.abs(np.diff(rgb, axis=1)).mean()
    assert tv < 0.2   # uniform-random colours give ~0.67


def test_deployment_bin_container_and_layout():
    from taichi_nerfs_b200.layout import make_hash_layout
    kat_lego.stage()
    emb = kat_lego.read_bin(os.path.join(kat_lego.REF_DIR, "hash_embedding.bin"))
    assert emb.dtype == np.float32 and emb.size == make_hash_layout(2 ** 21, 4, 32, 128, 4).total_param_size
    assert kat_lego.read_bin(os.path.join(kat_lego.REF_DIR, "sigma_weights.bin")).size == 512
    bits = kat_lego.read_bin(os.path.join(kat_lego.REF_DIR, "density_bitfield.bin")).view(np.uint8)
    assert np.array_equal(bits, np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"])
