"""The tri-plane model in the graph-captured training step (StaticTrainStep on a TriPlaneEncoder model) and the
device-counted table backward it runs (ngp_triplane_encode_bwd_dyn, csrc/triplane.cu).

Kernel: world positions with the AABB folded in, a device row count below n_max, NaN rows beyond the count, guard bands
around the table and the gradient, against the fp64 scatter of tests/triplane_ref.py; the inf flag; the static entry as
the NULL call of the same code.  The rows are ray runs (constant step sqrt(3)/1024 along a direction): long runs inside
one coarse cell, axis-aligned runs that end exactly on a cell boundary of level 0 and single-row rays, so that a kernel
that accumulates a run in registers has its flushes exercised.

Step: the comparators of tests/test_gpu_graph_step_grads.py, stage by stage on the step's own buffers, with the
tri-plane encoder's oracle (oracle/triplane.py) for the embedding and the whole gradient.

Inputs that terminate rays: the golden Lego bitfield, a U[0, 1) plane table (seed 11), init_weights_numpy(7) with
w1 x 4 and sigma's row of w2 replaced by 4 |row| (the embedding is a product of three features in [0, 1), all positive;
a signed row gives a median sigma below 1) and targets in [1.25, 2) (see _host_batch).  The oracle on the 2048 rays
of the first batch: 45 k rows, sigma up to 1.2e5, 578 rays terminate early, |dL/dsigma * sigma| <= 76 at loss scale 2^19.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import test_gpu_graph_step_grads as G
from triplane_ref import _check_triplane_scatter, _table_at
from triplane_ref import np_triplane_bwd_f64 as _BWD

THR = G.THR
N_RAYS = G.N_RAYS
CFG = dict(scale=0.5, max_res=1024, half=False, esf=0.0, bits="lego", spr=384, sampled=False)
FULL = dict(CFG, bits="full")
def np_triplane_bwd_f64(xn, table, dout, lay):
    return _BWD(xn, _table_at(table), dout, lay)


AABB = (-0.5, -0.5, -0.5, 1.0, 1.0, 1.0)
DT = 3 ** 0.5 / 1024


def _layout(F=4, max_res=1024):
    from taichi_nerfs_b200.layout import make_triplane_layout
    return make_triplane_layout(8, 16, max_res, F)


def _normalise(xw):
    """networks.py:144 in fp32, as load_position does with aabb6 = AABB."""
    return ((np.asarray(xw, np.float32) - np.float32(-0.5)) / np.float32(1.0)).astype(np.float32)


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib
    return _lib.load()


@pytest.fixture(autouse=True)
def _collect_after_each_test():
    """The steps built here own CUDA graphs; collect them when the test ends, not whenever the cyclic collector next
    runs (destroying a graph while a later test captures one invalidates that capture)."""
    yield
    import gc
    gc.collect()


# ---- kernel inputs ----------------------------------------------------------------------------------------------------
def ray_run_rows(seed=0):
    """World positions [n, 3] grouped as ray runs, in an arbitrary order of the runs."""
    rng = np.random.default_rng(seed)
    runs = []
    for _ in range(6):                                     # long runs inside one cell of level 0 (cell side 1/15)
        start = (rng.integers(2, 12, 3) + 0.2) / 15 - 0.5
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        runs.append(start + np.arange(24)[:, None] * DT * d)
    for axis in range(3):                                  # runs that end exactly on a cell boundary of level 0:
        for m in (5, 8, 13):                               # normalised x*15 + 0.5 = integer at the last row
            end = np.full(3, 0.31)
            end[axis] = (7 - 0.5) / 15
            d = np.eye(3)[axis]
            runs.append(end - 0.5 - np.arange(m)[::-1, None] * DT * d)
    for _ in range(40):                                    # ordinary rays across the box
        start = rng.random(3) - 0.5
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        runs.append(start + np.arange(int(rng.integers(2, 40)))[:, None] * DT * d)
    runs += [rng.random((1, 3)) - 0.5 for _ in range(17)]  # single-row rays
    order = rng.permutation(len(runs))
    return np.concatenate([runs[i] for i in order]).astype(np.float32)


def _kernel_case(F, seed=0):
    lay = _layout(F)
    rng = np.random.default_rng(100 + seed)
    xw = ray_run_rows(seed)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    dout = rng.normal(size=(xw.shape[0], lay.out_dim)).astype(np.float32)
    dout[rng.random(xw.shape[0]) < 0.15] = 0               # rows behind the termination point
    dout[:, 3 * 1] *= (rng.random(xw.shape[0]) < 0.5)      # and single zero columns
    return lay, xw, table, dout


GUARD = 1024          # floats on each side; a multiple of 4 keeps the inner pointer aligned to one entry
SENTINEL = np.float32(-7.25)


def check_bwd_dyn(got, guards_ok, lay, xw, table, dout, count, what):
    """Test 1's comparator: `got` the gradient buffer (prefill 0) after a backward on the first `count` rows of world
    positions xw."""
    assert guards_ok, f"{what}: a guard band was written"
    idx, ref, mag, cnt = np_triplane_bwd_f64(_normalise(xw[:count]), table, dout[:count], lay)
    return _check_triplane_scatter(got, np.zeros_like(got), idx, ref, mag, cnt, what)


def _run_bwd_dyn(lay, xw, table, dout, n_dev, use_aabb=True, found_inf=True, static=False):
    """Launch on guarded buffers.  Returns (gradient [P], guards intact, found_inf value)."""
    import torch
    from taichi_nerfs_b200._lib import check, load
    P = lay.total_param_size
    tbuf = torch.full((P + 2 * GUARD,), float("nan"), device="cuda")
    tbuf[GUARD:GUARD + P] = torch.from_numpy(table).cuda()
    gbuf = torch.full((P + 2 * GUARD,), float(SENTINEL), device="cuda")
    gbuf[GUARD:GUARD + P] = 0
    x, dy = torch.from_numpy(xw).cuda().contiguous(), torch.from_numpy(dout).cuda().contiguous()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())   # noqa: E731
    cl = lay.as_ctypes()
    tp, gp = C.c_void_p(tbuf.data_ptr() + 4 * GUARD), C.c_void_p(gbuf.data_ptr() + 4 * GUARD)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if static:
        check(load().ngp_triplane_encode_bwd(p(x), tp, p(dy), C.byref(cl), gp, x.shape[0], st))
    else:
        a6 = (C.c_float * 6)(*AABB) if use_aabb else None
        check(load().ngp_triplane_encode_bwd_dyn(p(x), tp, p(dy), C.byref(cl), gp, x.shape[0], p(nd), a6,
                                                 p(flag) if found_inf else None, st))
    torch.cuda.synchronize()
    g = gbuf.cpu().numpy()
    ok = bool((g[:GUARD] == SENTINEL).all() and (g[GUARD + P:] == SENTINEL).all())
    return g[GUARD:GUARD + P].copy(), ok, int(flag)


def _poisoned(xw, dout, count):
    xw, dout = xw.copy(), dout.copy()
    xw[max(count, 0):] = np.nan
    dout[max(count, 0):] = np.nan
    return xw, dout


@pytest.mark.gpu
@pytest.mark.parametrize("F", [2, 4])
def test_bwd_dyn_against_fp64(lib, F):
    lay, xw, table, dout = _kernel_case(F)
    n = xw.shape[0]
    for n_dev in (n - 37, 0, 1, n, n + 5, -3):
        count = min(max(n_dev, 0), n)
        xp, dp = _poisoned(xw, dout, count)
        got, ok, flag = _run_bwd_dyn(lay, xp, table, dp, n_dev)
        r = check_bwd_dyn(got, ok, lay, xw, table, dout, count, f"F={F} n_dev={n_dev}")
        assert flag == 0, (n_dev, flag)
        print(f"\n[bwd_dyn F={F} n_dev={n_dev}] rows {count} of {n}, err/bound max {r:.3f}")
    got, ok, flag = _run_bwd_dyn(lay, xw, table, dout, None)          # n_dev == NULL: n_max rows
    check_bwd_dyn(got, ok, lay, xw, table, dout, n, "n_dev NULL")


@pytest.mark.gpu
def test_bwd_dyn_inf_flag(lib):
    lay, xw, table, dout = _kernel_case(4, seed=1)
    n = xw.shape[0]
    count = n - 20
    live = int(np.flatnonzero((dout[:count] != 0).any(1))[4])
    for bad in (np.inf, np.nan):
        d = dout.copy()
        d[live, 5] = bad
        assert _run_bwd_dyn(lay, xw, table, d, count)[2] == 1, bad
        d = dout.copy()
        d[count + 2, 5] = bad                                          # the same value beyond the count
        got, ok, flag = _run_bwd_dyn(lay, xw, table, d, count)
        assert flag == 0
        check_bwd_dyn(got, ok, lay, xw, table, dout, count, "non-finite dout beyond the count")
    # an all-zero dout row whose corners are NaN in the table: nothing gathered, nothing scattered, nothing raised
    from triplane_ref import corner_entry, triplane_axes, triplane_ori
    d = dout.copy()
    d[live] = 0
    others = np.delete(np.arange(count), live)
    idx_others = np.concatenate([np_triplane_bwd_f64(_normalise(xw[others]), table, np.ones_like(dout[others]), lay)[0]])
    t = table.copy()
    _, q = triplane_axes(_normalise(xw[live:live + 1]), lay, 7)
    ori = [[triplane_ori(qb, lay.max_res) for qb in qk] for qk in q]
    e = int(corner_entry(lay, ori, 0, 0)[0])
    assert e not in set(idx_others.tolist()), "the chosen entry is shared with another row: pick another row"
    t[e] = np.nan
    got, ok, flag = _run_bwd_dyn(lay, xw, t, d, count)
    assert flag == 0 and ok and np.isfinite(got).all()


@pytest.mark.gpu
def test_static_entry_is_the_null_call_of_the_dyn_entry(lib):
    lay = _layout(4)
    rng = np.random.default_rng(5)
    xn = rng.random((48, 3), dtype=np.float32)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    dout = np.zeros((48, lay.out_dim), np.float32)
    for i in range(48):                                                # one live level per row
        dout[i, np.arange(4) * 8 + i % 8] = rng.normal(size=4)
    idx, ref, mag, cnt = np_triplane_bwd_f64(xn, table, dout, lay)
    assert cnt.max() == 1, "an entry receives two contributions: the atomic order would matter"
    a = _run_bwd_dyn(lay, xn, table, dout, None, static=True)
    b = _run_bwd_dyn(lay, xn, table, dout, None, use_aabb=False, found_inf=False)
    assert a[1] and b[1] and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))
    _check_triplane_scatter(a[0], np.zeros_like(a[0]), idx, ref, mag, cnt, "static entry")
    # many contributions per entry: both inside the fp64 bound
    lay, xw, table, dout = _kernel_case(4, seed=2)
    xn = _normalise(xw)
    idx, ref, mag, cnt = np_triplane_bwd_f64(xn, table, dout, lay)
    assert cnt.max() > 8
    for kw in (dict(static=True), dict(use_aabb=False, found_inf=False)):
        got, ok, _ = _run_bwd_dyn(lay, xn, table, dout, None, **kw)
        assert ok
        _check_triplane_scatter(got, np.zeros_like(got), idx, ref, mag, cnt, str(kw))


# ---- the step ---------------------------------------------------------------------------------------------------------
def _params():
    from bench import init_weights_numpy
    lay = _layout()
    _, _, ws = init_weights_numpy(7)
    ws = [w.copy() for w in ws]
    ws[0] *= 4
    ws[1][0] = 4 * np.abs(ws[1][0])
    return np.random.default_rng(11).random(lay.total_param_size, dtype=np.float32), ws


def _build(cfg=CFG, **trainer_kw):
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200.fused_mlp import mlp_weights
    from taichi_nerfs_b200.trainer import NGPTrainer
    table, ws = _params()
    m = NGP(scale=0.5, max_res=1024, half_opt=False, pos_encoder_type="triplane").cuda()
    bits = G._bitfield(cfg, m.density_bitfield.numel())
    with torch.no_grad():
        m.pos_encoder.plane_embedding.copy_(torch.from_numpy(table))
        for p, w in zip(mlp_weights(m), ws):
            p.copy_(torch.from_numpy(w))
        m.density_bitfield.copy_(torch.from_numpy(bits))
    return m, NGPTrainer(m, lr=1e-2, **trainer_kw), bits


def _host_batch(cfg, k):
    """G._host_batch with the targets moved to [1.25, 2): the head comparator bounds dL/drgb relative to itself, so a
    channel whose rendered colour lands within ~1e-4 of its target (with U[0, 1) targets: one ray of these 2048, on the
    oracle's own output too) has no admissible rounding; a target outside the colour range leaves no such channel."""
    o, d, gt, noise = G._host_batch(cfg, k)
    return o, d, (np.float32(1.25) + np.float32(0.75) * gt).astype(np.float32), noise


def _step(fs, k, cfg=CFG):
    import torch
    fs.step(*(torch.from_numpy(a).cuda() for a in _host_batch(cfg, k)))


def _snap(fs, m, bits):
    import torch
    s = G._snapshot(fs, m)
    torch.cuda.synchronize()
    s.update(bits=bits, flat_param=fs.tr.flat_param.detach().cpu().numpy().copy(),
             found_inf=int(fs.tr.found_inf), hyper=fs.hyper.detach().cpu().numpy().copy())
    return s


def _run_steps(n_steps, cfg=CFG, spr=None, **kw):
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, bits = _build(cfg)
    kw.setdefault("use_graph", True)
    kw.setdefault("overlap_optimizer", True)
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=spr or cfg["spr"], T_threshold=THR, **kw)
    assert fs.inf_at_source and tr._shadow is None and not fs.half and fs.emb.dtype == torch.float32
    snaps = []
    for k in range(n_steps):
        _step(fs, k, cfg)
        snaps.append(_snap(fs, m, bits))
    fs.flush()
    torch.cuda.synchronize()
    final = dict(flat_param=tr.flat_param.detach().cpu().numpy().copy(), kernels=fs.kernels_per_replay)
    del fs, tr, m
    torch.cuda.empty_cache()
    return snaps, final


@functools.lru_cache(maxsize=None)
def _runs():
    return _run_steps(2)


def check_triplane_fwd(snap, table):
    from oracle import triplane as OT
    ref = OT.triplane_encode_fwd(_normalise(snap["xyzs"]), table, _layout())
    same = (snap["emb"].view(np.uint32) == ref.view(np.uint32)).all(1)
    assert same.all(), f"tri-plane forward: {int((~same).sum())} of {same.size} rows differ"


def check_triplane_bwd(snap):
    """The plane-table gradient in flat_grad[:P] against the fp64 scatter of the step's own xyzs / demb."""
    P = snap["P"]
    got = snap["flat_grad"][:P]
    idx, ref, mag, cnt = np_triplane_bwd_f64(_normalise(snap["xyzs"]), snap["table"], snap["demb"], _layout())
    r = _check_triplane_scatter(got, np.zeros(P, np.float32), idx, ref, mag, cnt, "plane-table gradient")
    return dict(err_over_bound=r, entries=int(idx.size), k_max=int(cnt.max()))


def check_stages(snap, cfg=CFG):
    check_triplane_fwd(snap, snap["table"])
    st = dict(mlp_fwd=G.check_mlp_fwd(snap, snap["ws"]), head=G.check_head(snap, cfg, snap["gt"]))
    st["mlp_bwd"] = G.check_mlp_bwd(snap, snap["ws"])
    st["triplane_bwd"] = check_triplane_bwd(snap)
    return st


def check_end_to_end(snap, cfg=CFG):
    from oracle import triplane as OT
    om = OT.TriplaneOracleModel(_layout(), snap["table"], snap["ws"], snap["bits"])
    rgb_out, cache = OT.forward(om, snap["rays_o"], snap["rays_d"], snap["noise"], cfg["esf"], THR)
    _, g_table, g_mlp = OT.backward(om, cache, rgb_out, snap["gt"], snap["scale"])
    assert cache["S"] == snap["S"]
    st = G._grad_stats(snap["flat_grad"], snap["P"], g_table, g_mlp)
    G._assert_grad_stats(st, G.E2E_ALL_TABLE, G.E2E_ALL_BLOCK, "all-oracle chain")
    return st


def host_adam(param, grad, scale, lr, t=1, b1=0.9, b2=0.999, eps=1e-15):
    """One Adam step from zero moments in fp64 (train.py:143-156) on grad / scale."""
    g = grad.astype(np.float64) / scale
    m, v = (1 - b1) * g, (1 - b2) * g * g
    return param - lr * (m / (1 - b1 ** t)) / (np.sqrt(v / (1 - b2 ** t)) + eps)


@pytest.mark.gpu
@pytest.mark.parametrize("step", ["first", "steady"])
def test_triplane_graph_step_stages_against_fp64(step):
    snaps, final = _runs()
    snap = snaps[0 if step == "first" else 1]
    m = G.check_march(snap, CFG)
    assert m["cut"] == 0 and m["S"] == snap["counter"][0] < snap["cap"] and m["over32"] > 0
    assert snap["P"] == 12_582_912 and snap["found_inf"] == 0
    if step == "steady":
        prev = snaps[0]
        assert not np.array_equal(snap["table"], prev["table"]) and not np.array_equal(snap["ws"][1], prev["ws"][1])
        with pytest.raises(AssertionError):
            check_triplane_fwd(snap, prev["table"])
        # the parameters this step read are the first step's Adam on the first step's gradient (lr of iteration 0)
        want = host_adam(prev["flat_param"].astype(np.float64), prev["flat_grad"], prev["scale"], 1e-2)
        moved = prev["flat_grad"] != 0
        err = np.abs(snap["flat_param"] - want)
        assert (err[moved] <= 2e-6 * 1e-2 + 4 * G.U * np.abs(want[moved])).all(), float(err[moved].max())
        assert np.array_equal(snap["flat_param"][~moved], prev["flat_param"][~moved])
    st = check_stages(snap)
    assert st["head"]["terminated"] > 0 and st["head"]["ambiguous"] <= N_RAYS // 100, st["head"]
    G._report(f"triplane {step}", dict(march=m, **st))
    G._report(f"triplane {step} end to end", check_end_to_end(snap))


@pytest.mark.gpu
def test_triplane_graph_replay_equals_eager_enqueue():
    graph = _runs()[0]
    eager, _ = _run_steps(2, use_graph=False)
    for k, (a, b) in enumerate(zip(graph, eager)):
        # rows are reserved by atomics: compare ray by ray through rays_a
        assert np.array_equal(a["counter"], b["counter"])
        ia = np.concatenate([np.arange(s, s + c) for _, s, c in a["rays_a"]])
        ib = np.concatenate([np.arange(s, s + c) for _, s, c in b["rays_a"]])
        # the first step reads identical parameters: bit-identical up to the gradients' atomic order.  The second reads
        # what Adam made of two summation orders of the first gradient (an entry whose sum cancels can move the other
        # way): the march is still bit-identical, the embedding equal except for the rows that touch such an entry
        for name in ("xyzs", "emb", "sig", "rgbs", "demb") if k == 0 else ("xyzs",):
            x, y = a[name][ia], b[name][ib]
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (k, name)
        if k == 1:
            off = np.abs(a["emb"][ia] - b["emb"][ib]) > 1e-4 * np.abs(a["emb"][ia]) + 1e-7
            assert off.mean() < 1e-3, float(off.mean())
            continue
        assert np.array_equal(a["flat_grad"][a["P"]:] != 0, b["flat_grad"][b["P"]:] != 0)
        check_triplane_bwd(b)
        st = G._grad_stats(b["flat_grad"], b["P"], a["flat_grad"][:a["P"]], a["flat_grad"][a["P"]:a["P"] + G.MLP])
        assert st["table"]["max"] <= 1e-5, st          # two atomic orders of the same terms
        for i in range(1, 6):
            assert st[f"w{i}"]["max"] <= 1e-5, st


@pytest.mark.gpu
def test_triplane_capacity_overflow():
    """A fully occupied bitfield and a capacity a few thousand rows short of what the rays march."""
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from oracle import oracle as O
    o, d, gt, noise = _host_batch(FULL, 0)
    hits = O.ray_aabb_intersect(o, d, 0.5)
    S_all = O.raymarching_train(o, d, hits, np.full(128 ** 3 // 8, 255, np.uint8), noise, 1, 0.5, 0.0, 128, 1024)[5]
    spr = (S_all - 3000) // N_RAYS
    m, tr, bits = _build(FULL)
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=spr, T_threshold=THR, use_graph=True,
                         overlap_optimizer=True)
    cap = fs.cap
    assert cap < S_all <= cap + 3000 + N_RAYS
    # guard bands: the row buffers are exactly `cap` rows, so rows beyond it would be written into other allocations;
    # what can be checked here is that the rows at the end of the buffers are the truncated ray's and no more
    _step(fs, 0, FULL)
    snap = _snap(fs, m, bits)
    fs.flush()
    torch.cuda.synchronize()
    mm = G.check_march(snap, FULL)
    assert snap["counter"][0] == S_all > cap and mm["S"] == cap
    assert mm["partial"] == 1 and mm["cut"] > 1 and snap["counter"][1] == mm["cut"], mm
    st = check_stages(snap, FULL)
    G._report("triplane overflow", dict(march=mm, **st))


@pytest.mark.gpu
def test_triplane_overflowing_step_is_skipped():
    import torch
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, bits = _build()
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=CFG["spr"], T_threshold=THR, use_graph=True)
    assert fs.inf_at_source and float(fs.scale_state[0]) == 2.0 ** 19
    assert fs.kernels_per_replay > 0
    _step(fs, 0)
    i32 = lambda t: int(t.view(torch.int32))      # noqa: E731
    assert i32(fs.hyper[3:]) == 1 and int(tr.found_inf) == 0
    keep = [t.clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq)]
    with torch.no_grad():
        fs.scale_state[0] = 2.0 ** 126              # dL/drgb leaves fp16, dL/dout of the encoder is non-finite
    _step(fs, 1)
    torch.cuda.synchronize()
    for t, k in zip((tr.flat_param, tr.exp_avg, tr.exp_avg_sq), keep):
        assert torch.equal(t, k)                    # skipped: parameters and moments untouched
    assert i32(fs.hyper[3:]) == 1                   # Adam's step count did not advance
    assert float(fs.scale_state[0]) == 2.0 ** 125 and i32(fs.scale_state[1:]) == 0
    assert int(tr.found_inf) == 0                   # consumed and cleared by the optimizer
    assert float(tr.flat_grad.abs().max()) == 0     # the poisoned gradient is gone
    with torch.no_grad():
        fs.scale_state[0] = 2.0 ** 19
        fs.hyper[2] = 2.0 ** -19
    _step(fs, 2)
    torch.cuda.synchronize()
    assert i32(fs.hyper[3:]) == 2 and int(tr.found_inf) == 0 and float(fs.scale_state[0]) == 2.0 ** 19
    assert not torch.equal(tr.flat_param, keep[0]) and bool(torch.isfinite(tr.flat_param).all())


@pytest.mark.gpu
@pytest.mark.parametrize("w_d", [0.0, 1e-2])
def test_triplane_graph_step_equals_module_path(monkeypatch, w_d):
    """NGPTrainer.forward_backward on the same batch and noise: the MLP gradient and the plane-table gradient of the
    graph step ([with the distortion loss]); the loss as well."""
    import torch
    from modules.distortion import distortion_loss
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    o, d, gt, noise = (torch.from_numpy(a).cuda() for a in _host_batch(CFG, 0))
    m1, t1, _ = _build()
    monkeypatch.setattr(torch, "rand_like", lambda t, **k: noise.clone())
    extra = (lambda res: w_d * distortion_loss(res).mean()) if w_d > 0 else None
    loss1, _ = t1.forward_backward(o, d, gt, extra_loss=extra)
    monkeypatch.undo()
    torch.cuda.synchronize()
    g1 = t1.flat_grad.detach().cpu().numpy().copy()
    m2, t2, bits = _build()
    fs = StaticTrainStep(t2, N_RAYS, samples_per_ray_capacity=CFG["spr"], T_threshold=THR, use_graph=True,
                         overlap_optimizer=True, distortion_loss_w=w_d)
    loss2 = fs.step(o, d, gt, noise=noise)
    snap = _snap(fs, m2, bits)
    fs.flush()
    P = snap["P"]
    loss1, loss2 = float(loss1.detach()), float(loss2)
    assert abs(loss1 - loss2) <= 2e-3 * loss1, (loss1, loss2)
    # the module path runs autocast (fp16 sigma / rgb into its compositing): the bounds of the hash model's
    # module-path comparison (test_gpu_graph_step_grads.py: E2E_ALL_TABLE, E2E_ALL_BLOCK)
    st = G._grad_stats(snap["flat_grad"], P, g1[:P], g1[P:P + G.MLP])
    G._report(f"triplane graph step vs module path, w_d={w_d}", st)
    G._assert_grad_stats(st, G.E2E_ALL_TABLE, G.E2E_ALL_BLOCK, "module path")
    check_triplane_bwd(snap)


@pytest.mark.gpu
def test_triplane_sampled_steps_and_psnr_vs_teacher():
    """The arguments and the gate of tests/test_gpu_triplane.py::test_psnr_vs_teacher_triplane, through the graph."""
    import torch
    from taichi_nerfs_b200.psnr import train_vs_teacher
    r = train_vs_teacher(torch.device("cuda"), steps=1500, train_views=32, test_views=2, downsample=0.25,
                         pos_encoder_type="triplane", graph=True)
    if r is None:
        pytest.skip("teacher fixture not staged")
    print(f"\n[triplane graph psnr] {r['psnr']:.2f} dB, {r['rays_per_s'] / 1e6:.2f} M rays/s")
    assert r["path"] == "graph"
    assert r["psnr"] >= 24.7, r["psnr"]


@pytest.mark.gpu
def test_static_step_refusals():
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200._lib import NgpError
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    m, tr, _ = _build()
    StaticTrainStep(tr, 256, samples_per_ray_capacity=64, use_graph=False)
    m = NGP(scale=0.5, max_res=1024, half_opt=False, pos_encoder_type="triplane").cuda()
    m.xyz_encoder.net_width = 32                 # not the stock architecture
    with pytest.raises(NgpError):
        StaticTrainStep(NGPTrainer(m), 256)
    with pytest.raises(ValueError):
        m3, _, _ = _build(p2p_optimizer=True)    # the peer-memory optimizer stays refused


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_bwd_dyn_argument_validation_needs_no_gpu():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    L = _lib.load()
    cl = _layout().as_ctypes()
    buf = (C.c_float * 64)()
    a = C.addressof(buf)
    p = C.c_void_p(a)
    call = lambda *args: L.ngp_triplane_encode_bwd_dyn(*args)    # noqa: E731
    ok = (p, p, p, C.byref(cl), p)
    assert call(*ok, 0, None, None, None, None) == 0             # n_max == 0 returns before the pointer checks
    assert call(None, None, None, C.byref(cl), None, 0, None, None, None, None) == 0
    assert call(*ok, -1, None, None, None, None) != 0
    for k in (0, 1, 2, 4):
        args = list(ok)
        args[k] = None
        assert call(*args, 8, None, None, None, None) != 0, k
    assert call(p, p, p, None, p, 8, None, None, None, None) != 0
    assert call(p, p, p, C.byref(cl), C.c_void_p(a + 4), 8, None, None, None, None) != 0     # misaligned gradient
    assert b"aligned" in L.ngp_last_error()
    assert call(p, C.c_void_p(a + 4), p, C.byref(cl), p, 8, None, None, None, None) != 0     # misaligned table
    bad = _layout().as_ctypes()
    bad.feat_dim = 3
    assert call(p, p, p, C.byref(bad), p, 8, None, None, None, None) != 0
    bad = _layout().as_ctypes()
    bad.max_res = 1
    assert call(p, p, p, C.byref(bad), p, 8, None, None, None, None) != 0
    assert b"max_res" in L.ngp_last_error()


def _np_bwd(lay, xn, table, dout, run=None, drop_last_flush=False):
    """The table backward in numpy (fp64 sums rounded to fp32), optionally as a run-accumulating kernel of chunk
    `run` that forgets the last flush of every chunk."""
    from triplane_ref import corner_entry, corner_weight, triplane_axes, triplane_ori
    n, L, F = xn.shape[0], lay.levels, lay.feat_dim
    g = np.zeros(lay.total_param_size, np.float64)
    dy_all = dout.reshape(n, F, L).astype(np.float64)
    cols = np.arange(F)
    for level in range(L):
        a, q = triplane_axes(xn, lay, level)
        ori = [[triplane_ori(qb, lay.max_res) for qb in qk] for qk in q]
        e = [[corner_entry(lay, ori, fd, c) for c in range(4)] for fd in range(3)]
        w = [[corner_weight(a, fd, c).astype(np.float64) for c in range(4)] for fd in range(3)]
        lf = np.zeros((3, n, F))
        for fd in range(3):
            for c in range(4):
                lf[fd] += w[fd][c][:, None] * table[e[fd][c][:, None] + cols]
        dy = dy_all[:, :, level]
        live = (dy != 0).any(1)
        for fd in range(3):
            o1, o2 = [k for k in range(3) if k != fd]
            keep = live.copy()
            if drop_last_flush:      # the contributions still in registers when a chunk ends are lost
                cell = np.stack([e[fd][c] for c in range(4)], 1)
                for c0 in range(0, n, run):
                    rows_ = [i for i in range(c0, min(c0 + run, n)) if live[i]]
                    if rows_:
                        last = cell[rows_[-1]]
                        for i in rows_[::-1]:
                            if not (cell[i] == last).all():
                                break
                            keep[i] = False
            for c in range(4):
                v = (w[fd][c][:, None] * dy * lf[o1] * lf[o2])[keep]
                np.add.at(g, (e[fd][c][keep][:, None] + cols).reshape(-1), v.reshape(-1))
    return g.astype(np.float32)


@pytest.mark.parametrize("fault", [None, "ignores_aabb6", "reads_a_row_beyond_the_count", "drops_the_last_flush"])
def test_bwd_dyn_comparator_rejects_faulty_backwards(fault):
    lay = _layout(4, max_res=256)
    rng = np.random.default_rng(3)
    xw = ray_run_rows(3)
    table = rng.random(lay.total_param_size, dtype=np.float32)
    dout = rng.normal(size=(xw.shape[0], lay.out_dim)).astype(np.float32)
    count = xw.shape[0] - 11
    if fault is None:
        got = _np_bwd(lay, _normalise(xw[:count]), table, dout[:count])
    elif fault == "ignores_aabb6":
        got = _np_bwd(lay, xw[:count], table, dout[:count])
    elif fault == "reads_a_row_beyond_the_count":
        got = _np_bwd(lay, _normalise(xw[:count + 1]), table, dout[:count + 1])
    else:
        got = _np_bwd(lay, _normalise(xw[:count]), table, dout[:count], run=8, drop_last_flush=True)
    if fault is None:
        check_bwd_dyn(got, True, lay, xw, table, dout, count, "numpy restatement")
        with pytest.raises(AssertionError):
            check_bwd_dyn(got, False, lay, xw, table, dout, count, "guard band written")
    else:
        with pytest.raises(AssertionError):
            check_bwd_dyn(got, True, lay, xw, table, dout, count, fault)
