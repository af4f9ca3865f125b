"""The gradients of the graph-captured training step (taichi_nerfs_b200/fast_step.py: StaticTrainStep with
use_graph=True, overlap_optimizer=True, the mode bench.py measures), stage by stage on the step's own buffers.

Each stage is judged against a reference computed from the GPU's own inputs to that stage, so that one fp16 rounding
flip upstream is never held to a downstream bound:

1. march: hits and every ray's rows bit-exact against the oracle; rays_a tiles the rows (and, on capacity overflow,
   exactly one ray straddles the end of the buffers and keeps the samples that fit);
2. hash forward: bit-exact against the oracle on the table the step read;
3. MLP forward: sigma within the flip model of tests/mlp_tolerance.py, rgb within 4 fp16 ulp;
4. ray head: dL/dsigma, dL/drgb, opacity, rgb and the loss against fp64 compositing, the termination index of every
   ray accepted only inside the fp32 error window of the threshold (tests/composite_ref.py);
5. MLP backward: dL/demb and the weight gradient against the oracle (the error model of
   tests/test_gpu_parity.py::test_mlp_bwd_tcgen05_matches_oracle, constants measured on the step's rows);
6. hash backward: the table gradient against the fp64 scatter bound of tests/hash_ref.py, through the L2-sized level
   groups with a device row count below the capacity.

Then the whole gradient against the all-oracle chain (oracle/train_step.py), and the MLP gradient of the module path
(NGPTrainer.forward_backward).  The first step replays the "first" graph (forward + backward), the second the
"steady" one (Adam of the first step beside the second step's march), which must read the parameters that update
wrote.  The CPU tests at the end feed every comparator the oracle's own outputs, unmodified and with the faults a
looser check lets through.

Inputs that terminate rays: the golden Lego bitfield with init_weights_numpy(7), the table x 1e5 and sigma's row of
w2 x 2 (2048 rays of make_rays(seed=3): 45 k rows, 119 rays terminate early, 459 have more than 32 samples).
"""
import ctypes as C
import functools

import numpy as np
import pytest

from composite_ref import U, _check_composite_bwd, kernel_termination, np_composite_f64, termination_window
from hash_ref import _check_scatter, _level_slice, _normalise, np_hash_bwd_f64
from mlp_tolerance import check_sigma

THR = 1e-4
N_RAYS = 2048
MLP = 9408                                                 # w1 | w2 | w3 | w4 | w5 after the table in flat_grad
MLP_BLOCKS = np.cumsum([0, 2048, 1024, 2048, 4096, 192])
RGB_TOL = 4 * 2.0 ** -11                                   # 4 fp16 ulp in [0.5, 1)

CONFIGS = {
    "lego_half": dict(scale=0.5, max_res=1024, half=True, esf=0.0, bits="lego", spr=512, sampled=False),
    "lego_half_sampled": dict(scale=0.5, max_res=1024, half=True, esf=0.0, bits="lego", spr=512, sampled=True),
    # fp32 table and embedding, loss scale 2^19; 384 samples per ray keep the capacity below 2^20: one launch
    "lego_fp32": dict(scale=0.5, max_res=1024, half=False, esf=0.0, bits="lego", spr=384, sampled=False),
    # 6 cascades, exp_step_factor 1/256, background 0, max_res 4096
    "garden_half": dict(scale=16.0, max_res=4096, half=True, esf=1 / 256, bits="random", spr=512, sampled=False,
                        radius=3.0),
}
# fully occupied: 1,068,551 rows for the 2048 rays, ~20 k more than the 2^20 rows of capacity
OVERFLOW = dict(scale=0.5, max_res=1024, half=True, esf=0.0, bits="full", spr=512, sampled=False)


# ---- inputs ---------------------------------------------------------------------------------------------------------
def _layout(cfg):
    from taichi_nerfs_b200.layout import make_hash_layout
    return make_hash_layout(2 ** 19, 16, 16, cfg["max_res"], 2)


def _params(cfg):
    """(table [entries, 2] fp32, MLP weights): init_weights_numpy(7), table x 1e5, sigma's row of w2 x 2."""
    from bench import init_weights_numpy
    _, table, ws = init_weights_numpy(7, max_res=cfg["max_res"])
    ws[1] = ws[1].copy()
    ws[1][0] *= 2
    return (table * 1e5).astype(np.float32), ws


def _bitfield(cfg, size):
    if cfg["bits"] == "lego":
        import os
        from conftest import GOLDEN
        return np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"].copy()
    if cfg["bits"] == "full":
        return np.full(size, 255, np.uint8)
    rng = np.random.default_rng(5)       # ~30 % of the bytes occupied, as test_static_step_other_configs
    return ((rng.random(size) < 0.3) * rng.integers(1, 256, size)).astype(np.uint8)


def _host_batch(cfg, k):
    from oracle.train_step import make_rays
    o, d = make_rays(N_RAYS, seed=3 + k, radius=cfg.get("radius", 1.4))
    rng = np.random.default_rng(30 + k)
    return o, d, rng.random((N_RAYS, 3), dtype=np.float32), rng.random(N_RAYS, dtype=np.float32)


def _cascades(cfg):
    return 1 if cfg["scale"] <= 0.5 else 6


def _l2_groups(lay, n_max):
    """Level groups the step's table backward launches: the plan of ngp_hash_bwd_level_groups at the device's L2
    size, one group for launches of fewer than 2^20 rows."""
    import torch
    from taichi_nerfs_b200._lib import load
    if n_max < 1 << 20:
        return [0, lay.levels]
    bounds = (C.c_int32 * 17)()
    g = load().ngp_hash_bwd_level_groups(C.byref(lay.as_ctypes()), 0, lay.levels,
                                         torch.cuda.get_device_properties(0).L2_cache_size, bounds)
    assert g >= 1
    return list(bounds)[:g + 1]


# ---- running the step and reading its buffers -----------------------------------------------------------------------
def _snapshot(fs, m):
    """Every buffer of the last replay, on the host.  Rows at or beyond min(counter[0], capacity) are stale and are
    not read.  The parameters are those the replay read: the current fp16 shadow (or fp32 table) and fp32 MLP
    weights; the update of this step is still pending."""
    import torch
    from taichi_nerfs_b200.fused_mlp import mlp_weights
    torch.cuda.synchronize()
    cnt = fs.counter.cpu().numpy().copy()
    S = int(min(max(int(cnt[0]), 0), fs.cap))
    rows = lambda t: t[:S].detach().cpu().numpy().copy()       # noqa: E731
    full = lambda t: t.detach().cpu().numpy().copy()           # noqa: E731
    snap = {k: rows(getattr(fs, k)) for k in ("xyzs", "dirs", "deltas", "ts", "emb", "sig", "rgbs", "dsig", "drgbs",
                                              "demb")}
    snap.update({k: full(getattr(fs, k)) for k in ("hits", "rays_a", "rays_o", "rays_d", "gt", "noise", "loss_sum",
                                                   "opacity", "rgb")})
    snap.update(counter=cnt, S=S, cap=fs.cap, P=fs.P, flat_grad=full(fs.tr.flat_grad),
                scale=float(fs.scale_state[0]), table=full(fs._table()).reshape(-1),
                ws=[full(w) for w in mlp_weights(m)], half=fs.half, n_max=fs.cap)
    return snap


def _build(cfg, params=None):
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200.fused_mlp import mlp_weights
    from taichi_nerfs_b200.trainer import NGPTrainer
    table, ws = _params(cfg) if params is None else params
    m = NGP(scale=cfg["scale"], max_res=cfg["max_res"], half_opt=cfg["half"]).cuda()
    assert m.cascades == _cascades(cfg)
    bits = _bitfield(cfg, m.density_bitfield.numel())
    with torch.no_grad():
        ht = m.pos_encoder.hash_table
        ht.copy_(torch.from_numpy(table).reshape(ht.shape))
        for p, w in zip(mlp_weights(m), ws):
            p.copy_(torch.from_numpy(w))
        m.density_bitfield.copy_(torch.from_numpy(bits))
    return m, NGPTrainer(m, lr=1e-2), bits


def _run_steps(cfg, n_steps):
    """n_steps replays of the benchmark's mode; a snapshot after each, before anything applies its update."""
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, bits = _build(cfg)
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=cfg["spr"], exp_step_factor=cfg["esf"],
                         T_threshold=THR, use_graph=True, overlap_optimizer=True)
    if cfg["sampled"]:
        from datasets.synthetic import SyntheticLego
        ds = SyntheticLego(n_images=6, img_wh=(64, 64), focal=88.9, batch_size=N_RAYS, seed=2).to("cuda")
        ds.build_image_bank()
        fs.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=1234)
    snaps = []
    for k in range(n_steps):
        assert fs.pending == (k > 0)            # "first" graph, then "steady"
        if cfg["sampled"]:
            fs.step_sampled()
        else:
            o, d, gt, noise = _host_batch(cfg, k)
            fs.step(*(torch.from_numpy(a).cuda() for a in (o, d, gt, noise)))
        snaps.append(_snapshot(fs, m))
        assert fs.pending
    fs.flush()
    del fs, tr, m
    torch.cuda.empty_cache()
    for s in snaps:
        s["bits"] = bits
    return snaps


@functools.lru_cache(maxsize=None)
def _runs(name):
    return _run_steps(CONFIGS[name], 2)


# ---- the stage comparators (numpy: the CPU tests feed them the oracle's outputs) -------------------------------------
def check_march(snap, cfg):
    """Stage 1.  Returns (S, rays cut short, rays truncated inside their block, rays over 32 samples)."""
    from oracle import oracle as O
    o, d, noise, bits = snap["rays_o"], snap["rays_d"], snap["noise"], snap["bits"]
    hits = O.ray_aabb_intersect(o, d, cfg["scale"])
    assert np.array_equal(snap["hits"].view(np.uint32), hits.view(np.uint32)), "ray_aabb_intersect"
    ra_ref, xyzs, dirs, deltas, ts, S_all = O.raymarching_train(o, d, hits, bits, noise, _cascades(cfg), cfg["scale"],
                                                                cfg["esf"], 128, 1024)
    n, cap = o.shape[0], snap["cap"]
    ra, full = snap["rays_a"].astype(np.int64), ra_ref[:, 2].astype(np.int64)
    assert np.array_equal(ra[:, 0], np.arange(n)), "rays_a[:, 0] is not the ray index"
    keep = ra[:, 2]
    assert int(snap["counter"][0]) == S_all, (snap["counter"], S_all)           # every ray reserves its full count
    cut = keep != full
    assert int(snap["counter"][1]) == int(cut.sum()), (snap["counter"], int(cut.sum()))
    assert (keep >= 0).all() and (keep <= full).all(), "a ray owns more rows than it marched"
    partial = np.flatnonzero((keep > 0) & cut)
    assert partial.size <= 1, f"{partial.size} rays straddle the end of the buffers"
    assert (ra[keep == 0, 1] == 0).all(), "a ray without rows has a non-zero start"
    live = np.flatnonzero(keep > 0)
    order = live[np.argsort(ra[live, 1], kind="stable")]
    starts, counts = ra[order, 1], keep[order]
    S = min(S_all, cap)
    assert snap["S"] == S
    assert (starts.size == 0 or starts[0] == 0) and np.array_equal(starts[1:], np.cumsum(counts)[:-1]) \
        and int(counts.sum()) == S, "the kept blocks do not tile [0, min(counter, capacity))"
    idx = np.concatenate([np.arange(ra[r, 1], ra[r, 1] + keep[r]) for r in live])
    ref_idx = np.concatenate([np.arange(ra_ref[r, 1], ra_ref[r, 1] + keep[r]) for r in live])   # the first `keep`
    for name, ref in (("xyzs", xyzs), ("dirs", dirs), ("deltas", deltas), ("ts", ts)):
        assert np.array_equal(snap[name][idx].view(np.uint32), ref[ref_idx].view(np.uint32)), name
    return dict(S=S, cut=int(cut.sum()), partial=int(partial.size), over32=int((keep > 32).sum()))


def check_hash_fwd(snap, cfg, table):
    """Stage 2: emb bit-exact against the oracle on `table`, the table the step read."""
    from oracle import oracle as O
    ref = O.hash_encode_fwd(_normalise(snap["xyzs"], cfg["scale"]), table, _layout(cfg))
    got = snap["emb"]
    assert got.dtype == ref.dtype
    bits = np.uint16 if got.dtype == np.float16 else np.uint32
    same = (got.view(bits) == ref.view(bits)).all(1)
    assert same.all(), f"hash forward: {int((~same).sum())} of {same.size} rows differ"


def check_mlp_fwd(snap, ws):
    """Stage 3.  Returns the largest sigma error in fp16 ulp of h0 and the largest rgb error."""
    from oracle import oracle as O
    sig_ref, rgb_ref = O.mlp_fwd(snap["emb"], snap["dirs"], ws)
    u = check_sigma(snap["sig"], sig_ref, snap["emb"], ws)
    e_rgb = float(np.abs(snap["rgbs"].astype(np.float32) - rgb_ref.astype(np.float32)).max())
    assert e_rgb <= RGB_TOL, e_rgb
    return dict(sigma_ulp_max=u, rgb_max=e_rgb)


def _stats(err, scale):
    e = np.abs(err) / scale
    return dict(max=float(e.max()), p999=float(np.percentile(e, 99.9)), median=float(np.median(e)))


def check_head(snap, cfg, gt):
    """Stage 4 on the GPU's sig / rgbs / deltas / rays_a.  The termination index of every ray is the kernel's own
    (read from where its gradients become 0) and must lie inside the fp32 window of the threshold."""
    sig, rgbs, deltas, ts, ra = snap["sig"], snap["rgbs"], snap["deltas"], snap["ts"], snap["rays_a"]
    n, S = ra.shape[0], sig.size
    bg = 1.0 if cfg["esf"] == 0 else 0.0
    n_lo, n_hi, n64 = termination_window(sig, deltas, ra, THR)
    n_k = kernel_termination(snap["dsig"], snap["drgbs"], ra)
    bad = np.flatnonzero((n_k < n_lo) | (n_k > n_hi))
    assert bad.size == 0, (f"{bad.size} rays stop outside the fp32 window of the threshold, e.g. ray {bad[0]}: "
                           f"kernel {n_k[bad[0]]}, window [{n_lo[bad[0]]}, {n_hi[bad[0]]}], fp64 {n64[bad[0]]}")
    ambiguous = n_lo < n_hi
    assert not ((n_k != n64) & ~ambiguous).any()
    z, zs = np.zeros(n), np.zeros(S)
    fwd = np_composite_f64(sig, rgbs, deltas, ts, ra, THR, z, z, np.zeros((n, 3)), zs, n_active=n_k)
    out = fwd["rgb"] + bg * (1 - fwd["op"])[:, None]
    dd = out - gt.astype(np.float64)
    g = snap["scale"] * 2 * dd / (3 * n)
    ref = np_composite_f64(sig, rgbs, deltas, ts, ra, THR, -bg * g.sum(1), z, g, zs, n_active=n_k)
    _check_composite_bwd(snap["dsig"], snap["drgbs"], ref, True, "ray head")
    k = fwd["kray"]
    assert (np.abs(snap["opacity"] - fwd["op"]) <= 8 * k * U * fwd["op"] + 1e-30).all(), "opacity"
    e_out = 8 * k[:, None] * U * (np.abs(out) + 2)
    assert (np.abs(snap["rgb"] - out) <= e_out).all(), "rgb"
    loss = (dd ** 2).sum()
    assert abs(float(snap["loss_sum"][0]) - loss) <= (2 * np.abs(dd) * e_out).sum() + 16 * n * U * loss, "loss_sum"
    counts = np.zeros(n, np.int64)
    counts[ra[:, 0]] = ra[:, 2]
    return dict(terminated=int((n_k < counts).sum()), over32=int((counts > 32).sum()),
                ambiguous=int(ambiguous.sum()), chose_other_than_fp64=int((n_k != n64).sum()),
                dsig=_stats(snap["dsig"] - ref["dsig"], np.abs(ref["dsig"]).max()))


# Error model of the MLP backward on the step's rows (tests/test_gpu_parity.py::test_mlp_bwd_tcgen05_matches_oracle).
# Every intermediate gradient rounds to fp16 on both sides and the tensor core sums K in another order: the bulk agrees
# to a few 1e-7 of the tensor's max; ReLU-mask flips (a pre-activation within an ulp of 0) switch whole paths.
# Measured on an H100 over the eight first / steady steps and the overflow step (the largest of each):
MLP_DEMB_P999 = 2e-6        # of max |demb|; measured 2.0e-7
MLP_DEMB_MAX = 5e-3         # measured 2.6e-3 (garden_half steady): mask flips
MLP_BLOCK_MAX = 2e-3        # of each block's max |dW|; measured 5.2e-4
MLP_GW_MEDIAN = 5e-5        # median relative error of the dW entries above 5 % of the max; measured 5.2e-6


def check_mlp_bwd(snap, ws):
    """Stage 5 on the GPU's emb / dirs / dsig / drgbs."""
    from oracle import oracle as O
    P = snap["P"]
    demb_ref, gw_ref = O.mlp_bwd(snap["emb"], snap["dirs"], ws, snap["dsig"], snap["drgbs"])
    demb, demb_ref = snap["demb"].astype(np.float32), demb_ref.astype(np.float32)
    gw = snap["flat_grad"][P:P + MLP]
    scale = np.abs(demb_ref).max()
    assert scale > 0
    err = np.abs(demb - demb_ref)
    st = dict(demb=_stats(err, scale))
    assert st["demb"]["p999"] <= MLP_DEMB_P999, st
    assert st["demb"]["max"] <= MLP_DEMB_MAX, st
    for i, (a, b) in enumerate(zip(MLP_BLOCKS[:-1], MLP_BLOCKS[1:])):
        ref = gw_ref[a:b]
        assert np.abs(ref).max() > 0, f"w{i + 1}: empty gradient block"
        st[f"w{i + 1}"] = _stats(gw[a:b] - ref, np.abs(ref).max())
        assert st[f"w{i + 1}"]["max"] <= MLP_BLOCK_MAX, (i, st)
    big = np.abs(gw_ref) > 0.05 * np.abs(gw_ref).max()
    st["gw_big_median_rel"] = float(np.median(np.abs(gw[big] - gw_ref[big]) / np.abs(gw_ref[big])))
    assert st["gw_big_median_rel"] < MLP_GW_MEDIAN, st
    return st


def check_hash_bwd(snap, cfg):
    """Stage 6 on the GPU's xyzs / demb: the fp64 scatter bound over every level (prefill 0)."""
    lay = _layout(cfg)
    P = snap["P"]
    got = snap["flat_grad"][:P]
    ref, mag, cnt = np_hash_bwd_f64(_normalise(snap["xyzs"], cfg["scale"]), snap["demb"], lay, snap["half"],
                                    range(lay.levels))
    _check_scatter(got, np.zeros(P, np.float32), ref, mag, cnt, 0, P, "table gradient")
    return _stats(got - ref, np.abs(ref).max())


def check_stages(snap, cfg, table=None, ws=None, gt=None):
    """Stages 2-6; the parameters and targets default to those the step read."""
    table = snap["table"] if table is None else table
    ws = snap["ws"] if ws is None else ws
    gt = snap["gt"] if gt is None else gt
    check_hash_fwd(snap, cfg, table)
    st = dict(mlp_fwd=check_mlp_fwd(snap, ws), head=check_head(snap, cfg, gt))
    st["mlp_bwd"] = check_mlp_bwd(snap, ws)
    st["hash_bwd"] = check_hash_bwd(snap, cfg)
    return st


# Whole gradient against the all-oracle chain (oracle/train_step.py) on the same rays, noise, targets and parameters,
# relative to each tensor's max.  Measured on an H100, lego_half, 2048 rays: the table 8.2e-5 on the first step but
# 1.38e-3 on the steady step (p99.9 2.0e-7: a few entries), the MLP blocks up to 5.2e-4 (w1, steady).  The steady
# step's outliers come from the MLP backward: stage 5 on the same buffers measures dL/demb at 2.1e-3 and w1 at 5.1e-4
# of max, with its bulk at 7e-8, and the error is unchanged when the oracle composites the GPU's own sigma / rgb.
# These are ReLU-mask flips (a pre-activation within an fp16 ulp of 0), which the stage-5 error model admits.  So the
# north-star 1e-3 on the table's max holds on the first step but not on every step, and the bound here is 2e-3.
E2E_ALL_TABLE = 2e-3
E2E_ALL_TABLE_P999 = 1e-5
E2E_ALL_BLOCK = 2e-3        # module path (smoke recipe): w1 2.1e-4


def _grad_stats(fg, P, g_table, g_mlp):
    st = dict(table=_stats(fg[:P] - g_table, np.abs(g_table).max()))
    for i, (a, b) in enumerate(zip(MLP_BLOCKS[:-1], MLP_BLOCKS[1:])):
        st[f"w{i + 1}"] = _stats(fg[P + a:P + b] - g_mlp[a:b], np.abs(g_mlp[a:b]).max())
    return st


def _assert_grad_stats(st, table_max, block_max, what):
    assert st["table"]["max"] <= table_max, (what, st)
    for i in range(1, 6):
        assert st[f"w{i}"]["max"] <= block_max, (what, i, st)


def check_end_to_end(snap, cfg):
    from oracle import train_step as TS
    lay, P = _layout(cfg), snap["P"]
    om = TS.OracleModel(lay, snap["table"].astype(np.float32), snap["ws"], snap["bits"], scale=cfg["scale"],
                        cascades=_cascades(cfg), half=snap["half"])
    rgb_out, cache = TS.forward(om, snap["rays_o"], snap["rays_d"], snap["noise"], cfg["esf"], THR)
    _, g_table, g_mlp = TS.backward(om, cache, rgb_out, snap["gt"], snap["scale"])
    assert cache["S"] == snap["S"]
    st = _grad_stats(snap["flat_grad"], P, g_table, g_mlp)
    _assert_grad_stats(st, E2E_ALL_TABLE, E2E_ALL_BLOCK, "all-oracle chain")
    assert st["table"]["p999"] <= E2E_ALL_TABLE_P999, st
    return st


def _report(what, st):
    print(f"\n[{what}] {st}")


# ---- GPU: the four configurations, first and steady step ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,step", [(c, s) for c in CONFIGS for s in ("first", "steady")])
def test_graph_step_stages_against_fp64(name, step):
    cfg = CONFIGS[name]
    snaps = _runs(name)
    snap = snaps[0 if step == "first" else 1]
    m = check_march(snap, cfg)
    assert m["cut"] == 0 and snap["counter"][1] == 0 and m["S"] == snap["counter"][0] < snap["cap"]
    assert m["over32"] > 0, "no ray runs the head's multi-chunk path"
    if step == "steady":
        # the step read the parameters the first step's update wrote (the shadow / table and the MLP weights)
        prev = snaps[0]
        assert not np.array_equal(snap["table"], prev["table"]) and not np.array_equal(snap["ws"][1], prev["ws"][1])
        with pytest.raises(AssertionError):
            check_hash_fwd(snap, cfg, prev["table"])
    st = check_stages(snap, cfg)
    assert st["head"]["terminated"] > 0, "no ray terminates early"
    assert st["head"]["ambiguous"] <= N_RAYS // 100, st["head"]
    # the table backward the step ran: L2-sized level groups with the device row count below the capacity
    groups = _l2_groups(_layout(cfg), snap["n_max"])
    if snap["n_max"] >= 1 << 20:
        assert len(groups) > 2 and snap["counter"][0] < snap["n_max"], (groups, snap["counter"])
    else:
        assert name == "lego_fp32" and groups == [0, 16]
    _report(f"{name} {step}", dict(march=m, **st, level_groups=groups))


@pytest.mark.gpu
@pytest.mark.parametrize("step", ["first", "steady"])
def test_graph_step_gradient_equals_oracle_chain(step):
    snap = _runs("lego_half")[0 if step == "first" else 1]
    _report(f"lego_half {step} end to end", check_end_to_end(snap, CONFIGS["lego_half"]))


@pytest.mark.gpu
def test_graph_step_capacity_overflow_trains_on_truncated_rays():
    """A fully occupied bitfield marches ~20 k rows more than the 2^20 of capacity: exactly one ray keeps the samples
    that fit, the rays after it own no rows, and stages 2-6 are as exact on that layout as without overflow."""
    import torch
    snap = _run_steps(OVERFLOW, 1)[0]
    torch.cuda.empty_cache()
    m = check_march(snap, OVERFLOW)
    assert snap["counter"][0] > snap["cap"] == 1 << 20
    assert m["partial"] == 1 and m["cut"] > 1, m
    st = check_stages(snap, OVERFLOW)
    assert st["head"]["terminated"] > 0 and st["head"]["over32"] > 0
    _report("overflow", dict(march=m, **st))


@pytest.mark.gpu
@pytest.mark.parametrize("recipe", ["smoke", "terminating"])
def test_module_path_mlp_gradient_equals_oracle(monkeypatch, recipe):
    """NGPTrainer.forward_backward (the autograd path train.py uses by default): the MLP gradient, block by block, and
    the table gradient against the all-oracle chain on the same rays, with zero marching noise."""
    import torch
    from oracle import train_step as TS
    cfg = dict(CONFIGS["lego_half"])
    if recipe == "smoke":        # __graft_entry__.smoke(): table x 1e3, no ray terminates
        from bench import init_weights_numpy
        _, table, ws = init_weights_numpy(7)
        table = (table * 1e3).astype(np.float32)
    else:
        table, ws = _params(cfg)
    m, tr, bits = _build(cfg, (table, ws))
    o, d, gt, _ = _host_batch(cfg, 0)
    monkeypatch.setattr(torch, "rand_like", lambda t, **k: torch.zeros_like(t))
    loss, res = tr.forward_backward(*(torch.from_numpy(a).cuda() for a in (o, d, gt)))
    monkeypatch.undo()
    torch.cuda.synchronize()
    P = m.pos_encoder.total_param_size
    fg = tr.flat_grad.detach().cpu().numpy()
    om = TS.OracleModel(_layout(cfg), table, ws, bits, half=True)
    rgb_out, cache = TS.forward(om, o, d, np.zeros(N_RAYS, np.float32))
    _, g_table, g_mlp = TS.backward(om, cache, rgb_out, gt, float(tr.scale_state[0]))
    assert int(res["rm_samples"]) == cache["S"]
    st = _grad_stats(fg, P, g_table, g_mlp)
    _report(f"module path {recipe}", st)
    _assert_grad_stats(st, E2E_ALL_TABLE, E2E_ALL_BLOCK, "module path")
    assert st["table"]["p999"] <= E2E_ALL_TABLE_P999, st


# ---- CPU: every comparator accepts the oracle's outputs and rejects the faults --------------------------------------
CPU_RAYS = 256


def _oracle_snapshot(cfg, table, ws, bits, o, d, gt, noise, loss_scale, cap=None, network=True, seed=0):
    """What the step's buffers hold after one replay, computed by the oracle: rows reserved per ray in a random
    order (the march's atomics), the ray straddling `cap` keeping what fits, the network on min(S, cap) rows."""
    from oracle import oracle as O
    lay, n = _layout(cfg), o.shape[0]
    hits = O.ray_aabb_intersect(o, d, cfg["scale"])
    ra_ref, xyzs, dirs, deltas, ts, S_all = O.raymarching_train(o, d, hits, bits, noise, _cascades(cfg), cfg["scale"],
                                                                cfg["esf"], 128, 1024)
    cap = S_all if cap is None else cap
    rays_a = np.zeros((n, 3), np.int32)
    rays_a[:, 0] = np.arange(n)
    S = min(S_all, cap)
    buf = {k: np.zeros((S,) + a.shape[1:], np.float32) for k, a in (("xyzs", xyzs), ("dirs", dirs),
                                                                     ("deltas", deltas), ("ts", ts))}
    s0, cut = 0, 0
    for r in np.random.default_rng(seed).permutation(n):
        full, st = int(ra_ref[r, 2]), int(ra_ref[r, 1])
        keep = full if s0 + full <= cap else max(0, min(full, cap - s0))
        cut += keep != full
        rays_a[r, 1:] = (s0 if keep > 0 else 0, keep)
        for k, a in (("xyzs", xyzs), ("dirs", dirs), ("deltas", deltas), ("ts", ts)):
            buf[k][s0:s0 + keep] = a[st:st + keep]
        s0 += full
    half = cfg["half"]
    tab = table.reshape(-1).astype(np.float16 if half else np.float32)
    snap = dict(buf, hits=hits, rays_a=rays_a, rays_o=o, rays_d=d, gt=gt, noise=noise, bits=bits, S=S, cap=cap,
                counter=np.array([S_all, cut], np.int32), P=lay.total_param_size, half=half, table=tab, ws=ws,
                scale=float(loss_scale), n_max=cap)
    if not network:
        return snap
    xn = _normalise(snap["xyzs"], cfg["scale"])
    emb = O.hash_encode_fwd(xn, tab, lay)
    sig, rgbs = O.mlp_fwd(emb, snap["dirs"], ws)
    _, op, _, rgb, _ = O.composite_train_fwd(sig, rgbs, snap["deltas"], snap["ts"], rays_a, THR)
    bg = np.float32(1.0 if cfg["esf"] == 0 else 0.0)
    out = (rgb + bg * (1 - op)[:, None]).astype(np.float32)
    diff = out - gt
    g_rgb = (np.float32(loss_scale) * 2.0 * diff / np.float32(3 * n)).astype(np.float32)
    g_op = (-bg * g_rgb.sum(1)).astype(np.float32)
    dsig, drgbs = O.composite_train_bwd(g_op, np.zeros(n, np.float32), g_rgb, np.zeros(S, np.float32), sig, rgbs,
                                        snap["deltas"], snap["ts"], rays_a, THR)
    demb, gw = O.mlp_bwd(emb, snap["dirs"], ws, dsig, drgbs)
    g_table = O.hash_encode_bwd(xn, demb, lay)
    snap.update(emb=emb, sig=sig, rgbs=rgbs, dsig=dsig, drgbs=drgbs, demb=demb, opacity=op, rgb=out,
                loss_sum=np.array([(diff.astype(np.float32) ** 2).sum()], np.float32),
                flat_grad=np.concatenate([g_table, gw]))
    return snap


def _cpu_inputs(cfg, bits_kind="lego"):
    from oracle.train_step import make_rays
    c = dict(cfg, bits=bits_kind)
    o, d = make_rays(CPU_RAYS, seed=3)
    rng = np.random.default_rng(30)
    gt, noise = rng.random((CPU_RAYS, 3), dtype=np.float32), rng.random(CPU_RAYS, dtype=np.float32)
    size = 128 ** 3 // 8 * _cascades(c)
    return c, _bitfield(c, size), o, d, gt, noise


@pytest.fixture(scope="module")
def cpu_step(oracle):
    """The oracle's step on 256 rays at the parameters after one oracle Adam step ("current") and before it
    ("previous"): the buffers a correct step leaves, and those of a step that read stale parameters."""
    from oracle import train_step as TS
    cfg, bits, o, d, gt, noise = _cpu_inputs(CONFIGS["lego_half"])
    table, ws = _params(cfg)
    lay = _layout(cfg)
    om = TS.OracleModel(lay, table, ws, bits, half=True)
    rgb_out, cache = TS.forward(om, o, d, noise)
    _, g_table, g_mlp = TS.backward(om, cache, rgb_out, gt, 65536.0)
    prev = (om.shadow.copy(), [w.copy() for w in om.ws])
    assert TS.adam(om, g_table, g_mlp, 1e-2, 65536.0)
    cur = (om.shadow.astype(np.float32), [w.copy() for w in om.ws])
    snap = _oracle_snapshot(cfg, cur[0], cur[1], bits, o, d, gt, noise, 65536.0)
    stale = _oracle_snapshot(cfg, prev[0].astype(np.float32), prev[1], bits, o, d, gt, noise, 65536.0)
    return cfg, snap, stale


def test_comparators_accept_the_oracles_step(cpu_step):
    cfg, snap, _ = cpu_step
    m = check_march(snap, cfg)
    assert m["cut"] == 0 and m["over32"] > 0
    st = check_stages(snap, cfg)
    assert st["head"]["terminated"] > 0
    check_end_to_end(snap, cfg)


def _mutated(snap, **kw):
    s = dict(snap)
    s.update(kw)
    return s


def _first_level_group(cfg):
    """The first level group of the table backward at an 80 GB H100's 50 MiB of L2."""
    from taichi_nerfs_b200 import _lib, build
    build.build()
    lay = _layout(cfg)
    bounds = (C.c_int32 * 17)()
    g = _lib.load().ngp_hash_bwd_level_groups(C.byref(lay.as_ctypes()), 0, lay.levels, 50 << 20, bounds)
    assert g > 1
    return _level_slice(lay, bounds[0], bounds[1])


@pytest.mark.parametrize("fault", ["table_grad_x2", "level_group_scattered_twice"])
def test_table_gradient_comparators_reject(cpu_step, fault):
    cfg, snap, _ = cpu_step
    fg = snap["flat_grad"].copy()
    if fault == "table_grad_x2":
        fg[:snap["P"]] *= 2
    else:
        lo, hi = _first_level_group(cfg)
        fg[lo:hi] *= 2
    bad = _mutated(snap, flat_grad=fg)
    with pytest.raises(AssertionError):
        check_hash_bwd(bad, cfg)
    with pytest.raises(AssertionError):
        check_end_to_end(bad, cfg)


def test_head_comparator_rejects_dsigma_off_by_one_percent(cpu_step):
    cfg, snap, _ = cpu_step
    with pytest.raises(AssertionError):
        check_head(_mutated(snap, dsig=(snap["dsig"] * np.float32(1 + 1e-2)).astype(np.float32)), cfg, snap["gt"])


def test_head_comparator_rejects_swapped_targets(cpu_step):
    """The step's buffers computed with two rays' targets swapped, judged with the targets the step was given."""
    cfg, snap, _ = cpu_step
    ra = snap["rays_a"]
    a, b = ra[ra[:, 2] > 0, 0][:2]
    gt = snap["gt"].copy()
    gt[[a, b]] = gt[[b, a]]
    swapped = _oracle_snapshot(cfg, snap["table"].astype(np.float32), snap["ws"], snap["bits"], snap["rays_o"],
                               snap["rays_d"], gt, snap["noise"], snap["scale"])
    check_head(swapped, cfg, gt)
    with pytest.raises(AssertionError):
        check_head(swapped, cfg, snap["gt"])


@pytest.mark.parametrize("stage", ["hash_fwd", "mlp_fwd", "mlp_bwd"])
def test_stage_comparators_reject_stale_parameters(cpu_step, stage):
    """The buffers of a step that read the parameters from before the previous Adam step, judged with the current
    ones (the steady step's snapshot)."""
    cfg, snap, stale = cpu_step
    with pytest.raises(AssertionError):
        if stage == "hash_fwd":
            check_hash_fwd(stale, cfg, snap["table"])
        elif stage == "mlp_fwd":
            check_mlp_fwd(stale, snap["ws"])
        else:
            check_mlp_bwd(stale, snap["ws"])


def test_march_comparator_checks_the_truncated_ray(oracle):
    """Capacity overflow laid out as the march lays it out: accepted as is, rejected when the straddling ray keeps one
    sample too many (its block then runs past the capacity) or a later ray keeps rows."""
    cfg, bits, o, d, gt, noise = _cpu_inputs(OVERFLOW, "full")
    table, ws = _params(cfg)
    whole = _oracle_snapshot(cfg, table, ws, bits, o, d, gt, noise, 65536.0, network=False)
    S_all = whole["S"]
    cap = S_all - 5000
    snap = _oracle_snapshot(cfg, table, ws, bits, o, d, gt, noise, 65536.0, cap=cap, network=False)
    m = check_march(snap, cfg)
    assert m["partial"] == 1 and m["cut"] > 1 and m["S"] == cap
    ra = snap["rays_a"]
    full = whole["rays_a"][:, 2]
    r = np.flatnonzero((ra[:, 2] > 0) & (ra[:, 2] < full))[0]
    plus = ra.copy()
    plus[r, 2] += 1
    with pytest.raises(AssertionError):
        check_march(_mutated(snap, rays_a=plus), cfg)
    later = ra.copy()
    d_ = np.flatnonzero((ra[:, 2] == 0) & (full > 0))[0]
    later[d_, 1:] = (ra[r, 1], 1)                      # a dropped ray claiming a row
    with pytest.raises(AssertionError):
        check_march(_mutated(snap, rays_a=later), cfg)
