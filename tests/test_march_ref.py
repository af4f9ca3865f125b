"""The CPU oracle's ray march against an independent restatement of the reference (tests/march_ref.py) at every cascade
setting the project ships or tests, on well-formed and edge rays; fp64 checks of its samples, shown to reject planted
mistakes; the end of rays the reference marches forever; and agreement of the occupancy-grid update's cell positions
with the march's cell lookup."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import march_ref as R

f32 = np.float32
G = 128
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (scale, cascades, exp_step_factor, occupancy): the configurations of tests/test_gpu_parity.py::MARCH_CFGS.
# cascades = 1 + ceil(log2(2 scale)) and esf = 1/256 for scale > 0.5, as the reference's train.py derives them.
CFGS = {
    "lego": (0.5, 1, 0.0, "lego"),
    "random": (0.5, 1, 0.0, "random"),
    "6casc_esf": (16.0, 6, 1 / 256, "random"),
    "3casc_sparse": (2.0, 3, 1 / 256, "sparse"),
    "5casc_scale8": (8.0, 5, 1 / 256, "random"),        # the scale README.md ships for real scenes
    "3casc_scale1.5": (1.5, 3, 1 / 256, "random"),      # top cascade bound 1.5 < 2: inexact 1/mip_bound
    "4casc_scale3": (3.0, 4, 1 / 256, "sparse"),
    "8casc_scale64": (64.0, 8, 1 / 256, "random"),
}


def _bits(occ, cascades, rng, lego):
    nbytes = cascades * G ** 3 // 8
    if occ == "lego":
        return lego
    if occ == "full":
        return np.full(nbytes, 255, np.uint8)
    if occ == "random":
        return rng.integers(0, 256, nbytes, dtype=np.uint8)
    return (rng.random(nbytes) < 0.02).astype(np.uint8) * rng.integers(1, 256, nbytes, dtype=np.uint8)


def _inputs(name, n, seed, rays_factory, lego_bitfield):
    """Camera rays (from outside the box at scale 0.5, inside it otherwise) followed by the edge rays, their march
    intervals, and the configuration's bitfield."""
    scale, casc, esf, occ = CFGS[name]
    rng = np.random.default_rng(seed)
    o, d = rays_factory(n, seed=seed, radius=1.4 if scale == 0.5 else 3.0)
    eo, ed, eh, _ = R.edge_rays(scale, seed=seed)
    o, d = np.concatenate([o, eo]), np.concatenate([d, ed])
    hits = np.concatenate([R.aabb(o[:n], d[:n], scale), eh])
    return o, d, hits, _bits(occ, casc, rng, lego_bitfield), rng


def _same(a, b):
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", list(CFGS))
def test_restatement_equals_oracle(oracle, rays_factory, lego_bitfield, name):
    """Training march (with and without jitter) and test march with its resume points: the oracle == the
    restatement, bit for bit, on camera rays and every edge ray."""
    scale, casc, esf, _ = CFGS[name]
    o, d, hits, bits, rng = _inputs(name, 400, 31, rays_factory, lego_bitfield)
    assert _same(oracle.ray_aabb_intersect(o, d, scale), R.aabb(o, d, scale))
    n = o.shape[0]
    for noise in (rng.random(n, dtype=f32), np.zeros(n, f32)):
        ra, xyzs, dirs, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, noise, casc, scale, esf, G, 1024)
        cnt, ray, r_ts, r_dl, r_xyz = R.march_train(o, d, hits, bits, casc, scale, esf, G, 1024, noise=noise)
        assert S > 1000
        assert np.array_equal(ra[:, 2], cnt)
        assert _same(ts, r_ts) and _same(deltas, r_dl) and _same(xyzs, r_xyz)
        assert np.array_equal(dirs, d[ray])
    alive = np.concatenate([rng.permutation(400)[:200], np.arange(400, n)]).astype(np.int64)   # every edge ray
    for m in (1, 33):
        h_ref = hits.copy()
        ri, valid, dl, tt, c = oracle.raymarching_test(o, d, h_ref, alive, bits, casc, scale, esf, G, m)
        r_c, r_t, r_d, r_h = R.march_test(o, d, hits, alive, bits, casc, scale, esf, G, m)
        assert np.array_equal(c, r_c)
        v = valid.astype(bool).reshape(-1, m)
        assert np.array_equal(v, np.arange(m)[None, :] < r_c[:, None])
        assert _same(tt.reshape(-1, m)[v], r_t[v]) and _same(dl.reshape(-1, m)[v], r_d[v])
        assert _same(h_ref, r_h)                                   # resume points


@pytest.mark.parametrize("name", list(CFGS))
def test_fp64_checks_hold_on_oracle(oracle, rays_factory, lego_bitfield, name):
    """Every sample the oracle emits, training and test march, passes the fp64 checks."""
    scale, casc, esf, _ = CFGS[name]
    o, d, hits, bits, rng = _inputs(name, 3000, 32, rays_factory, lego_bitfield)
    n = o.shape[0]
    for noise in (rng.random(n, dtype=f32), np.zeros(n, f32)):
        ra, xyzs, _, deltas, ts, S = oracle.raymarching_train(o, d, hits, bits, noise, casc, scale, esf, G, 1024)
        R.check_samples(o, d, hits, np.repeat(ra[:, 0], ra[:, 2]), ts, deltas, xyzs, bits, casc, scale, esf)
    alive = np.arange(n, dtype=np.int64)
    h = hits.copy()
    ri, valid, dl, tt, c = oracle.raymarching_test(o, d, h, alive, bits, casc, scale, esf, G, 64)
    v = valid.astype(bool)
    x = o[ri[v]] + tt[v][:, None] * d[ri[v]]                      # fp32 o + t d, as the module test loop forms it
    R.check_samples(o, d, hits, ri[v], tt[v], dl[v], x.astype(f32), bits, casc, scale, esf)


def _fault_probe(rays_factory):
    """Rays on which each planted fault shows: camera rays from outside a 1.5-scale, 3-cascade box with esf 1/256
    (the step reaches the faulty dt_max = scale/G past t = 3) and rays held on the planes +-0.5 and +-1 (max|x| an exact
    power of two, and at the + face the grid coordinate is clamped to G - 1), against a random bitfield."""
    scale, casc, esf = 1.5, 3, 1 / 256
    o, d = rays_factory(600, seed=33, radius=3.0)
    hits = R.aabb(o, d, scale)
    fo, fd, fh = [], [], []
    rng = np.random.default_rng(33)
    for a in (0.5, 1.0):
        for sg in (1.0, -1.0):
            for k in range(16):
                p = np.array([sg * a, *rng.uniform(-0.6 * a, -0.3 * a, 2)])
                q = rng.normal(size=2)
                q = np.abs(q) / np.linalg.norm(q)
                fo.append(p)
                fd.append([0.0, q[0], q[1]])
                fh.append([0.01, 0.8 * a])
    o = np.concatenate([o, np.asarray(fo, f32)])
    d = np.concatenate([d, np.asarray(fd, f32)])
    hits = np.concatenate([hits, np.asarray(fh, f32)])
    bits = rng.integers(0, 256, casc * G ** 3 // 8, dtype=np.uint8)
    return o, d, hits, bits, scale, casc, esf


@pytest.mark.parametrize("fault", R.FAULTS)
def test_fp64_checks_reject_planted_faults(oracle, rays_factory, fault):
    """A marcher with one planted mistake -- doubled mip_bound, swapped Morton axes, clamp at G, frexp without the
    power-of-two rule, dt_max = scale/G, no cascade offset -- fails the fp64 checks, which the correct restatement and
    the oracle pass on the same rays."""
    o, d, hits, bits, scale, casc, esf = _fault_probe(rays_factory)
    noise = np.random.default_rng(34).random(o.shape[0], dtype=f32)
    cnt, ray, ts, dl, xyz = R.march_train(o, d, hits, bits, casc, scale, esf, G, 1024, noise=noise)
    R.check_samples(o, d, hits, ray, ts, dl, xyz, bits, casc, scale, esf)
    ra, o_xyz, _, o_dl, o_ts, _ = oracle.raymarching_train(o, d, hits, bits, noise, casc, scale, esf, G, 1024)
    assert _same(o_ts, ts)
    cnt_f, ray_f, ts_f, dl_f, xyz_f = R.march_train(o, d, hits, bits, casc, scale, esf, G, 1024, noise=noise,
                                                    fault=fault)
    assert not (np.array_equal(cnt_f, cnt) and _same(ts_f, ts))
    with pytest.raises(AssertionError):
        R.check_samples(o, d, hits, ray_f, ts_f, dl_f, xyz_f, bits, casc, scale, esf)


def test_edge_rays_cover_what_they_name(lego_bitfield):
    """The edge rays do what their names say: binade boundaries at the named chunk lane, exact zeros at the origin
    rays, components at the -1e-3 threshold, and samples at max|x| = 0.5 / 1 on the power-of-two planes."""
    o, d, hits, names = R.edge_rays(16.0)
    dt = R.SQRT3_MAX_SAMPLES
    for i, nm in enumerate(names):
        if nm.startswith("binade"):
            B, lane = float(nm[6:].split("_")[0]), int(nm.split("lane")[1])
            chain = [hits[i, 0]]
            for _ in range(lane + 1):
                chain.append(f32(chain[-1] + dt))
            assert chain[lane] < B <= chain[lane + 1], nm
        if nm.startswith("through_origin"):
            assert not (o[i] + hits[i, 0] * d[i]).any(), nm
    thr = [d[i, 0] for i, nm in enumerate(names) if nm.startswith("dir_minus1e-3_")]
    assert f32(-1e-3) in thr and (np.asarray(thr) < f32(-1e-3)).any() and (np.asarray(thr) > f32(-1e-3)).any()
    full = np.full(6 * G ** 3 // 8, 255, np.uint8)
    cnt, ray, ts, dl, xyz = R.march_train(o, d, hits, full, 6, 16.0, 1 / 256, G, 1024)
    mx = np.abs(xyz).max(1)
    for a in (0.5, 1.0, 2.0):
        assert (mx == a).sum() > 100
    assert (mx == 0).any()                                         # the through-origin rays' first samples


_DEGENERATE = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from oracle import oracle as O
import march_ref as R
o, d, names = R.degenerate_rays()
out = {"aabb": O.ray_aabb_intersect(o, d, 0.5).tolist()}
hits = np.array([[0.01, np.inf]] * 3 + [R.aabb(o[3:], d[3:], 0.5)[0]], np.float32)   # [0.01, +inf), [0.01, 2e29)
for scale, casc, esf in ((0.5, 1, 0.0), (8.0, 5, 1 / 256)):
    for occ in (0, 255):
        bits = np.full(casc * 128 ** 3 // 8, occ, np.uint8)
        ra, xyzs, _, _, ts, S = O.raymarching_train(o, d, hits, bits, np.zeros(4, np.float32), casc, scale, esf, 128, 1024)
        h = hits.copy()
        _, _, _, tt, c = O.raymarching_test(o, d, h, np.arange(4), bits, casc, scale, esf, 128, 64)
        out[f"{scale}/{occ}"] = {"train": ra[:, 2].tolist(), "test": c.tolist(), "finite": bool(np.isfinite(ts).all())}
print(json.dumps(out))
"""


def test_degenerate_rays_end(oracle):
    """Zero or NaN direction, NaN origin, direction 1e-30: the reference never ends these rays.  The oracle's AABB
    test reports a miss for a far hit that is not finite, and its marches end every ray -- given the reference's
    intervals [0.01, +inf) and [0.01, 2e29) too -- with no sample in an empty grid and at most max_samples in a full
    one.  Run in a subprocess under a timeout, so that a march that does not end fails the test instead of hanging
    the suite.  The restatement, which follows the reference, reports them by exceeding its step budget."""
    try:
        p = subprocess.run([sys.executable, "-c", _DEGENERATE, ROOT], capture_output=True, text=True, timeout=120)
    except subprocess.TimeoutExpired:
        pytest.fail("the oracle's march did not end on a degenerate ray within 120 s")
    assert p.returncode == 0, p.stderr
    out = json.loads(p.stdout)
    o, d, _ = R.degenerate_rays()
    assert out["aabb"][:3] == [[-1.0, -1.0]] * 3                 # no finite far hit: a miss
    assert 1e29 < out["aabb"][3][1] < 1e30
    ref = R.aabb(o, d, 0.5)                                           # intersection.py:8-37 on these rays
    assert ref[0, 1] == np.inf and ref[3, 1] == f32(out["aabb"][3][1])
    for key in ("0.5/0", "8.0/0"):
        assert out[key]["train"] == [0, 0, 0, 0] and out[key]["test"] == [0, 0, 0, 0], (key, out[key])
    for key in ("0.5/255", "8.0/255"):
        assert max(out[key]["train"]) <= 1024 and max(out[key]["test"]) <= 64 and out[key]["finite"], (key, out[key])
    hits = np.array([[0.01, np.inf]] * 3 + [ref[3]], f32)
    empty = np.zeros(G ** 3 // 8, np.uint8)
    for i in range(4):
        with pytest.raises(R.StepBudgetExceeded):
            R.march_train(o[i:i + 1], d[i:i + 1], hits[i:i + 1], empty, 1, 0.5, 0.0, G, 1024, budget=2000)


@pytest.mark.parametrize("cascades,scale", [(5, 8.0), (6, 16.0), (3, 1.5)])
def test_grid_cells_land_where_drawn(oracle, cascades, scale):
    """Warm-up grid update (networks.py:168-179, 263-271): the position drawn for cell i of cascade c, looked up with
    the march's arithmetic at mip c (ray_march.py:51-60), lands in cell i -- except within the fp32 window of a cell
    face, where it may land in the neighbour across that face."""
    grid = np.zeros((cascades, G ** 3), f32)
    idx, xyz = oracle.grid_sample_cells(grid, scale, 0.01, True, 0, 0x5EED, 3)
    per = G ** 3
    checked = 0
    for c in range(cascades):
        sl = slice(c * per, (c + 1) * per)
        mb = np.fmin(f32(2.0 ** (c - 1)), f32(scale))
        v = f32(0.5) * (xyz[sl] * (f32(1) / mb) + f32(1)) * f32(G)
        u = np.fmin(np.fmax(v, f32(0)), f32(G - 1)).astype(np.int64)
        drawn = oracle.morton3d_invert(idx[sl]).astype(np.int64)
        diff = u - drawn
        near = np.abs(v - np.round(v)) <= 2.0 ** -21 * G             # the fp32 window of a face, in grid units
        ok = (diff == 0) | ((np.abs(diff) == 1) & near)
        assert ok.all(), (c, np.nonzero(~ok.all(1))[0][:5])
        assert (diff == 0).all(1).mean() > 0.999
        checked += per
    assert checked == cascades * per
