"""The voxel-grid model (`--model_name svox`) in the graph-captured training step (StaticTrainStep on a VoxelGrid), the
device-counted field backward it runs (ngp_voxel_bwd_dyn) and its optimizer pass over the node block B
(ngp_check_finite_voxel_block, ngp_adam_step_voxel_block_dyn; DESIGN.md §6b).

Block kernels: against the dense ngp_check_finite / ngp_adam_step_dyn bit for bit, over every element of both fields.
Backward: the fp64 comparator of tests/test_gpu_voxel_grid.py with the device row count at every edge.  Step: the
comparators of tests/test_gpu_graph_step_grads.py (march), tests/test_gpu_voxel_fp64.py (voxel forward and backward),
tests/test_gpu_graph_step_distortion.py (head, with fp32 colours and ReLU-zero samples, see _composite_f64_relu) and
tests/voxel_reg_ref.py (regularisers), on the step's own buffers; then the module path, replay against eager enqueue, overlap against sync, the region invariant, the
failure paths and training end to end.
"""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

import test_gpu_graph_step_grads as G
import test_gpu_voxel_fp64 as V
import voxel_reg_ref as RR
from taichi_nerfs_b200.layout import make_voxel_layout, voxel_reg_block

pytestmark = pytest.mark.gpu

DEV = "cuda"
THR = G.THR
N_RAYS = G.N_RAYS
CFG = dict(scale=0.5, esf=0.0, bits="lego", spr=384)
LAT = dict(grid_size=97, grid_radius=0.0125, sh_degree=2)      # B = 84^3 of 97^3 nodes: every face of B is inside
REG = (0.01, 0.01, 0.0)
I32 = lambda t: t.view(torch.int32)                              # noqa: E731


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(autouse=True)
def _collect_after_each_test():
    """The steps built here own CUDA graphs; collect them when the test ends (see test_gpu_triplane_graph_step.py)."""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


# ---- 1. the block kernels against the dense pass ---------------------------------------------------------------------
def _hyper(t=3, lr=1e-2, inv_scale=2.0 ** -19, b1=0.9, b2=0.999):
    h = torch.tensor([lr / (1 - b1 ** t), math.sqrt(1 - b2 ** t), inv_scale, 0.0], device=DEV)
    I32(h)[3] = t
    return h


def _block_state(shape, block, seed, outside=0.0):
    """param random everywhere; grad, exp_avg, exp_avg_sq random inside B and `outside` elsewhere."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    p = torch.randn(shape, device=DEV, generator=gen)
    st = [torch.full(shape, outside, device=DEV) for _ in range(3)]
    b = RR.block_of
    b(st[0], block).copy_(torch.randn(b(st[0], block).shape, device=DEV, generator=gen) * 2.0 ** 19)
    b(st[1], block).copy_(torch.randn(b(st[1], block).shape, device=DEV, generator=gen) * 1e-2)
    b(st[2], block).copy_(torch.rand(b(st[2], block).shape, device=DEV, generator=gen) * 1e-4)
    return [p] + st


def _dense(bufs, flag, hyper):
    p, g, m, v = bufs
    from taichi_nerfs_b200._lib import check, load
    check(load().ngp_adam_step_dyn(_p(p), _p(g), _p(m), _p(v), None, _p(flag), _p(hyper), 0.9, 0.999, 1e-15, 1,
                                   p.numel(), _st()))


def _blockwise(bufs, block, flag, hyper):
    from taichi_nerfs_b200 import ops
    p, g, m, v = bufs
    ops.adam_step_voxel_block(p, g, m, v, block, hyper, found_inf=flag)


@pytest.mark.parametrize("deg", [0, 1, 2])
@pytest.mark.parametrize("G_,radius,scale", [(256, 0.0125, 0.5), (97, 0.03, 0.5), (2, 0.3, 0.5), (97, 0.03, 2.0)])
def test_block_adam_equals_dense_adam(G_, radius, scale, deg):
    from taichi_nerfs_b200 import ops
    lay = make_voxel_layout(G_, radius, deg)
    block = voxel_reg_block(lay, scale)
    if scale == 2.0:
        assert block == (0, 0, 0, G_, G_, G_)          # the box leaves the lattice: B is the whole grid
    hyper = _hyper()
    for C_ in (3 * lay.sh_dim, 1):
        shape = (G_, G_, G_, C_)
        a = _block_state(shape, block, seed=G_ + C_)
        b = [t.clone() for t in a]
        flag = torch.zeros(1, device=DEV, dtype=torch.int32)
        ops.check_finite(a[1], flag)
        ops.check_finite_voxel_block(b[1], block, flag)
        assert int(flag) == 0
        _dense(a, flag, hyper)
        _blockwise(b, block, flag, hyper)
        for name, x, y in zip(("param", "grad", "exp_avg", "exp_avg_sq"), a, b):
            assert torch.equal(x, y), (name, C_)
        assert not bool(b[1].any())
        del a, b
    torch.cuda.empty_cache()


def test_block_kernels_flag_sentinels_and_nonfinite():
    from taichi_nerfs_b200 import ops
    lay = make_voxel_layout(97, 0.03, 2)
    block = voxel_reg_block(lay, 0.5)
    hyper = _hyper()
    shape = (97, 97, 97, 27)
    SENT = -7.25
    ref = _block_state(shape, block, seed=3, outside=SENT)
    inside = torch.zeros(shape[:3] + (1,), dtype=torch.bool, device=DEV)
    RR.block_of(inside, block).fill_(True)
    # sentinels outside B: bit-unchanged, inside B as the dense pass on zero-outside copies
    b = [t.clone() for t in ref]
    _blockwise(b, block, None, hyper)
    a = [torch.where(inside, t, torch.zeros_like(t)) if k else t.clone() for k, t in enumerate(ref)]
    _dense(a, None, hyper)
    for x, y, r in zip(a, b, ref):
        assert torch.equal(torch.where(inside, x, r), y)
    # a raised flag: nothing changes but the gradient inside B, which is zeroed
    b = [t.clone() for t in ref]
    flag = torch.ones(1, device=DEV, dtype=torch.int32)
    _blockwise(b, block, flag, hyper)
    for k in (0, 2, 3):
        assert torch.equal(b[k], ref[k])
    assert torch.equal(b[1], torch.where(inside, torch.zeros_like(ref[1]), ref[1]))
    # non-finite values: inside B (first, last and an interior node) raise the flag, outside B they do not
    lo, hi = block[:3], block[3:]
    for node, ch, want in (((lo[0], lo[1], lo[2]), 0, 1), ((hi[0] - 1, hi[1] - 1, hi[2] - 1), 26, 1),
                           (tuple((a + b) // 2 for a, b in zip(lo, hi)), 13, 1), ((lo[0] - 1, 50, 50), 3, 0),
                           ((50, 50, hi[2]), 0, 0)):
        for bad in (math.nan, math.inf, -math.inf):
            g = ref[1].clone()
            g[node + (ch,)] = bad
            flag = torch.zeros(1, device=DEV, dtype=torch.int32)
            ops.check_finite_voxel_block(g, block, flag)
            assert int(flag) == want, (node, ch, bad)


def test_block_adam_past_2_pow_31_floats():
    """A degree-2 field at G = 432 (2,176,782,336 floats) with B at the far corner: every offset passes 2^31.  The
    buffers are left uninitialised except B and a guard at the start of each (where an int32 wrap would land)."""
    free, _ = torch.cuda.mem_get_info()
    if free < 40 * 2 ** 30:
        pytest.skip(f"needs ~36 GB of device memory, {free / 2 ** 30:.1f} GB free")
    from taichi_nerfs_b200 import ops
    G_, C_ = 432, 27
    block = (427, 390, 401, 432, 432, 432)
    n = G_ ** 3 * C_
    assert ((427 * G_ + 390) * G_ + 401) * C_ > 2 ** 31            # B's first float
    bufs = [torch.empty((G_, G_, G_, C_), device=DEV) for _ in range(4)]
    small = _block_state((5, 42, 31, C_), (0, 0, 0, 5, 42, 31), seed=9)
    GUARD = 1 << 22
    for t, s in zip(bufs, small):
        RR.block_of(t, block).copy_(s)
        t.view(-1)[:GUARD] = -3.5
    hyper = _hyper()
    flag = torch.zeros(1, device=DEV, dtype=torch.int32)
    ops.check_finite_voxel_block(bufs[1], block, flag)
    assert int(flag) == 0
    _blockwise(bufs, block, flag, hyper)
    _dense(small, flag, hyper)
    for t, s in zip(bufs, small):
        assert torch.equal(RR.block_of(t, block), s)
        assert bool((t.view(-1)[:GUARD] == -3.5).all())
    assert n > 2 ** 31


# ---- 2. the device-counted backward ---------------------------------------------------------------------------------
def _dyn_as_static(extra, n_dev_of, flags):
    """A stand-in for ops.voxel_bwd that runs ngp_voxel_bwd_dyn on the rows padded with `extra` NaN rows and the count
    n_dev_of(n): the rows past the count must never be read."""
    from taichi_nerfs_b200 import ops
    dyn = ops.voxel_bwd_dyn

    def f(xyz, dirs, sigma, rgb, dsig, drgb, cl, dsh, dden, found_inf=None, mapping=0):
        n = xyz.shape[0]
        pad = lambda t: torch.cat([t, torch.full((extra,) + tuple(t.shape[1:]), math.nan, device=t.device)])  # noqa
        flag = torch.zeros(1, device=DEV, dtype=torch.int32)
        nd = torch.tensor([n_dev_of(n)], device=DEV, dtype=torch.int32)
        dyn(pad(xyz), pad(dirs), pad(sigma), pad(rgb), pad(dsig), pad(drgb), cl, dsh, dden, n_dev=nd, found_inf=flag)
        flags.append(int(flag))
    return f


@pytest.mark.parametrize("G_,deg", [(256, 2), (97, 0), (97, 1), (2, 2)])
def test_bwd_dyn_against_fp64(monkeypatch, G_, deg):
    import test_gpu_voxel_grid as VG
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(G_ * 10 + deg + 1)
    lay = make_voxel_layout(G_, VG._radius(G_), deg)
    xyz = VG._positions(rng, 20001, G_, lay)
    dirs = torch.from_numpy(rng.standard_normal((xyz.shape[0], 3)).astype(np.float32))
    sh, den = VG._fields(G_ * 10 + deg, G_, deg)
    flags = []
    # the count below n_max (NaN rows past it), equal to it, above it
    for extra, nd in ((37, lambda n: n), (0, lambda n: n), (0, lambda n: n + 5)):
        monkeypatch.setattr(ops, "voxel_bwd", _dyn_as_static(extra, nd, flags))
        VG._check_fwd_bwd(G_, deg, xyz, dirs, sh, den, ops.VOXEL_BWD_WARP)
    assert flags == [0, 0, 0]


def test_bwd_dyn_row_count_edges_inf_flag_and_null_count():
    from taichi_nerfs_b200 import ops
    lay = make_voxel_layout(16, 0.125, 2)
    cl = lay.as_ctypes()
    sh = torch.rand(16, 16, 16, 27, device=DEV)
    den = torch.rand(16, 16, 16, 1, device=DEV)
    x = torch.rand(500, 3, device=DEV) - 0.5
    d = torch.randn(500, 3, device=DEV)
    s, c = ops.voxel_fwd(x, d, sh, den, cl)
    ds, dc = torch.randn_like(s), torch.randn_like(c)

    def run(n_dev, dcol=dc, found=True):
        dsh, dden = torch.zeros_like(sh), torch.zeros_like(den)
        flag = torch.zeros(1, device=DEV, dtype=torch.int32)
        nd = None if n_dev is None else torch.tensor([n_dev], device=DEV, dtype=torch.int32)
        ops.voxel_bwd_dyn(x, d, s, c, ds, dcol, cl, dsh, dden, n_dev=nd, found_inf=flag if found else None)
        return dsh, dden, int(flag)

    for nd in (0, -3, -2 ** 31):
        dsh, dden, f = run(nd)
        assert not bool(dsh.any()) and not bool(dden.any()) and f == 0
    bad = dc.clone()
    bad[123, 1] = math.inf
    assert run(None, bad)[2] == 1 and run(124, bad)[2] == 1
    dsh, dden, f = run(123, bad)                     # the row is past the count: not read
    assert f == 0 and bool(torch.isfinite(dsh).all())
    # the static entry is the NULL call: one contribution per node makes the sums order-free, so bit for bit
    G_ = 97
    lay = make_voxel_layout(G_, 2.0 ** -5, 2)
    cl = lay.as_ctypes()
    sh = torch.rand(G_, G_, G_, 27, device=DEV) * 2 - 1
    den = torch.rand(G_, G_, G_, 1, device=DEV) * 2 - 1
    cells = torch.tensor([(i, j, k) for i in range(2, 90, 3) for j in range(5, 90, 29) for k in range(1, 90, 44)],
                         dtype=torch.float64)
    x = (lay.c_min + (cells + torch.rand(cells.shape, dtype=torch.float64) * 0.9 + 0.05) * lay.radius).float().to(DEV)
    d = torch.randn(x.shape[0], 3, device=DEV)
    s, c = ops.voxel_fwd(x, d, sh, den, cl)
    ds, dc = torch.randn_like(s), torch.randn_like(c)
    a = (torch.zeros_like(sh), torch.zeros_like(den))
    b = (torch.zeros_like(sh), torch.zeros_like(den))
    ops.voxel_bwd(x, d, s, c, ds, dc, cl, *a)
    ops.voxel_bwd_dyn(x, d, s, c, ds, dc, cl, *b)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and bool(a[0].any())


# ---- the step ---------------------------------------------------------------------------------------------------------
def _build(lat=LAT, voxel_reg=None, seed=5, den_range=(-10.0, 50.0), bits="lego", **trainer_kw):
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.trainer import NGPTrainer
    m = VoxelGrid(scale=0.5, **lat).to(DEV)
    b = G._bitfield(dict(bits=bits), m.density_bitfield.numel())
    gen = torch.Generator(device=DEV).manual_seed(seed)
    with torch.no_grad():
        m.sh_fields.uniform_(-1, 1, generator=gen)
        m.density_fields.uniform_(*den_range, generator=gen)
        m.density_bitfield.copy_(torch.from_numpy(b))
    return m, NGPTrainer(m, lr=1e-2, voxel_reg=voxel_reg, **trainer_kw), b


def _batch(k, dev=True):
    """Rays of test_gpu_graph_step_grads._host_batch with targets in [1.25, 2) (see test_gpu_triplane_graph_step.py)."""
    o, d, gt, noise = G._host_batch(CFG, k)
    gt = (np.float32(1.25) + np.float32(0.75) * gt).astype(np.float32)
    return tuple(torch.from_numpy(a).to(DEV) for a in (o, d, gt, noise)) if dev else (o, d, gt, noise)


def _snap(fs, bits):
    torch.cuda.synchronize()
    cnt = fs.counter.cpu().numpy().copy()
    S = int(min(max(int(cnt[0]), 0), fs.cap))
    rows = lambda t: t[:S].detach().cpu().numpy().copy()       # noqa: E731
    full = lambda t: t.detach().cpu().numpy().copy()           # noqa: E731
    s = {k: rows(getattr(fs, k)) for k in ("xyzs", "dirs", "deltas", "ts", "sig", "rgbs", "dsig", "drgbs")}
    s.update({k: full(getattr(fs, k)) for k in ("hits", "rays_a", "rays_o", "rays_d", "gt", "noise", "loss_sum",
                                               "opacity", "rgb")})
    m = fs.model
    s.update(counter=cnt, S=S, cap=fs.cap, bits=bits, scale=float(fs.scale_state[0]),
             flat_grad=full(fs.tr.flat_grad), flat_param=full(fs.tr.flat_param), found_inf=int(fs.tr.found_inf),
             sh=m.sh_fields.detach().cpu().clone(), den=m.density_fields.detach().cpu().clone())
    return s


def _run_steps(n_steps, lat=LAT, voxel_reg=None, w_d=0.0, **kw):
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, bits = _build(lat, voxel_reg)
    kw.setdefault("use_graph", True)
    kw.setdefault("overlap_optimizer", True)
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=CFG["spr"], T_threshold=THR, distortion_loss_w=w_d, **kw)
    assert fs.vox and not fs.inf_at_source and fs.emb is None and fs.rgbs.dtype == torch.float32
    snaps, losses = [], []
    for k in range(n_steps):
        losses.append(float(fs.step(*_batch(k))))
        snaps.append(_snap(fs, bits))
    fs.flush()
    torch.cuda.synchronize()
    final = dict(flat_param=tr.flat_param.detach().cpu().numpy().copy(), losses=losses, kernels=fs.kernels_per_replay,
                 block=fs.block)
    del fs, tr, m
    return snaps, final


@functools.lru_cache(maxsize=None)
def _runs(w_d=0.0, reg=False):
    return _run_steps(2, voxel_reg=REG if reg else None, w_d=w_d)


def _fields_of(flat, m_shape_sh, m_shape_den):
    n = int(np.prod(m_shape_sh))
    off = n + (-n) % 4
    return (torch.from_numpy(flat[:n].reshape(m_shape_sh)),
            torch.from_numpy(flat[off:off + int(np.prod(m_shape_den))].reshape(m_shape_den)))


def _composite_f64_relu(*args, **kw):
    """composite_ref.np_composite_f64 with the conditioning factor k = N + 4 / min a of every ray taken over the
    composited samples with a > 0.

    Why: the voxel grid's sigma is ReLU(density), so a sample can have sigma = 0 exactly (the hash model's TruncExp
    never gives 0).  There a = 0 in fp64, so 4 / min a = inf, and the comparator's drgb bound for that ray becomes
    8 k u |drgb_ref| = inf * 0 = NaN at every sample of the ray with w = 0, which no value satisfies: that is what
    rejected the step's head.  Such a sample carries no error at all: the kernel computes a = 1 - expf(-0 * delta) = 0
    exactly, so w = a T = 0, dL/drgb = 0 and T_{s+1} = T_s exactly.  The factor 4 / a bounds the relative error of w
    that the absolute fp32 error of a causes, so only samples with a > 0 enter the minimum."""
    out = _ORIG_COMPOSITE(*args, **kw)
    sig, deltas, rays_a = args[0], args[2], args[4]
    a = -np.expm1(-(sig.astype(np.float64) * deltas.astype(np.float64)))
    for r, s0, cnt in rays_a:
        if cnt == 0:
            continue
        sl = slice(s0, s0 + cnt)
        live = a[sl][out["active"][sl] & (a[sl] > 0)]
        out["kray"][r] = cnt + (4.0 / live.min() if live.size else 0.0)
        out["k"][sl] = out["kray"][r]
    return out


import composite_ref as _CR                                     # noqa: E402
_ORIG_COMPOSITE = _CR.np_composite_f64


def check_svox_head(snap, w_d, faults=()):
    """The head on the step's buffers against fp64 (test_gpu_graph_step_distortion.check_head_dist, which with w_d = 0
    is the plain head's comparator), fp32 colours (half=False), with _composite_f64_relu."""
    import test_gpu_graph_step_distortion as D
    got = (snap["loss_sum"][0], snap["opacity"], snap["rgb"], snap["dsig"], snap["drgbs"])
    args = (snap["sig"], snap["rgbs"], snap["deltas"], snap["ts"], snap["rays_a"], snap["gt"], 1.0, snap["scale"], w_d,
            THR, False, f"svox step head w_d={w_d}")
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(D, "np_composite_f64", _composite_f64_relu)
        h = D.check_head_dist(got, *args, faults=faults)
    ra = snap["rays_a"]
    n_k = _CR.kernel_termination(snap["dsig"], snap["drgbs"], ra)
    counts = np.zeros(ra.shape[0], np.int64)
    counts[ra[:, 0]] = ra[:, 2]
    act = h["fwd"]["active"]
    return dict(terminated=int((n_k < counts).sum()), relu_zero_samples=int((snap["sig"][act] == 0).sum()),
                k_max=float(h["fwd"]["kray"].max()))


def check_voxel_stages(snap, lay, w_d=0.0, reg=None):
    """Voxel forward, head, backward [+ the regularisers' addition] on the step's own buffers."""
    xyz, dirs = torch.from_numpy(snap["xyzs"]), torch.from_numpy(snap["dirs"])
    sh, den = snap["sh"], snap["den"]
    ref = V.fwd_ref(xyz, dirs, sh, den, lay)
    st = dict(fwd=V.check_fwd(torch.from_numpy(snap["sig"]), torch.from_numpy(snap["rgbs"]), ref, "step forward"))
    st["head"] = check_svox_head(snap, w_d)
    dsig, drgb = torch.from_numpy(snap["dsig"]), torch.from_numpy(snap["drgbs"])
    nodes, want, tol = V.bwd_ref(xyz, dirs, sh, den, lay, dsig, drgb, ref, torch.from_numpy(snap["sig"]))
    dsh, dden = _fields_of(snap["flat_grad"], sh.shape, den.shape)
    block = voxel_reg_block(lay, 0.5)
    Gn = lay.grid
    ijk = torch.stack([nodes // (Gn * Gn), nodes // Gn % Gn, nodes % Gn], 1)
    inB = ((ijk >= torch.tensor(block[:3])) & (ijk < torch.tensor(block[3:]))).all(1)
    assert not bool((want[~inB] != 0).any()), "a sample's gradient reaches a node outside B"
    outside = torch.ones(sh.shape[:3], dtype=torch.bool)
    RR.block_of(outside, block).fill_(False)
    assert not bool(dsh[outside].any()) and not bool(dden[outside].any()), "a gradient float outside B"
    if reg is None:
        assert V._written_outside(dsh, dden, nodes) == 0
        st["bwd"] = V.check_bwd(V._kernel_grad_rows(dsh, dden, nodes), want, tol, "step backward")
        return st
    # regularisers: out = backward part + scale * fp64 regulariser gradient, within both bounds
    lo = torch.tensor(block[:3])
    bi = ijk[inB] - lo
    D3 = sh.shape[-1]
    pre = [torch.zeros(RR.block_of(t, block).shape, dtype=torch.float64) for t in (sh, den)]
    tb = [torch.zeros_like(p) for p in pre]
    for k, sl in ((0, slice(0, D3)), (1, slice(D3, D3 + 1))):
        pre[k][bi[:, 0], bi[:, 1], bi[:, 2]] = want[inB][:, sl]
        tb[k][bi[:, 0], bi[:, 1], bi[:, 2]] = tol[inB][:, sl]
    _, gS, gP, A_sh, A_den = RR.reference(RR.block_of(sh, block), RR.block_of(den, block), reg)
    worst = 0.0
    for name, out, p, g, A, t in (("sh", dsh, pre[0], gS, A_sh, tb[0]), ("density", dden, pre[1], gP, A_den, tb[1])):
        err = (RR.block_of(out, block).double() - (p + snap["scale"] * g)).abs()
        b = RR.bound(p, g, A, snap["scale"]) + t
        assert bool((err <= b).all()), (name, float((err - b).max()))
        worst = max(worst, float((err / b.clamp(min=1e-300)).max()))
    st["bwd_plus_reg"] = worst
    return st


def _lay(lat=LAT):
    return make_voxel_layout(lat["grid_size"], lat["grid_radius"], lat["sh_degree"])


@pytest.mark.parametrize("w_d,reg", [(0.0, False), (1e-2, False), (0.0, True)])
def test_svox_graph_step_stages_against_fp64(w_d, reg):
    snaps, final = _runs(w_d, reg)
    for k, snap in enumerate(snaps):
        m = G.check_march(snap, CFG)
        assert m["cut"] == 0 and m["S"] == snap["counter"][0] < snap["cap"] and m["over32"] > 0
        assert snap["found_inf"] == 0
        st = check_voxel_stages(snap, _lay(), w_d, REG if reg else None)
        # the buffers have ReLU-zero samples inside composited runs (the case _composite_f64_relu handles), and rays
        # that terminate early
        assert st["head"]["relu_zero_samples"] > 0 and st["head"]["terminated"] > 0, st["head"]
        if w_d > 0:   # the distortion's dL/dw is visible at this bound: the same buffers fail without it
            with pytest.raises(AssertionError):
                check_svox_head(snap, w_d, faults=("no_gw",))
        G._report(f"svox step {k} w_d={w_d} reg={reg}", dict(march=m, **st))
    # the second step read the first step's update: Adam's first step from zero moments on the first gradient
    prev, snap = snaps
    g = prev["flat_grad"].astype(np.float64) / prev["scale"]
    want = prev["flat_param"] - 1e-2 * g / (np.abs(g) + 1e-15)
    moved = prev["flat_grad"] != 0
    err = np.abs(snap["flat_param"] - want)
    assert (err[moved] <= 2e-6 * np.abs(want[moved]) + 1e-7).all(), float(err[moved].max())
    assert np.array_equal(snap["flat_param"][~moved], prev["flat_param"][~moved])


def test_svox_graph_replay_equals_eager_and_overlap_equals_sync():
    graph, gfin = _runs()
    for kw in (dict(use_graph=False), dict(overlap_optimizer=False)):
        other, ofin = _run_steps(2, **kw)
        for k, (a, b) in enumerate(zip(graph, other)):
            assert np.array_equal(a["counter"], b["counter"]), kw
            ia = np.concatenate([np.arange(s, s + c) for _, s, c in a["rays_a"]])
            ib = np.concatenate([np.arange(s, s + c) for _, s, c in b["rays_a"]])
            assert np.array_equal(a["xyzs"][ia].view(np.uint32), b["xyzs"][ib].view(np.uint32)), (kw, k)
            if k == 0:           # identical parameters: the forward and the head are bit-identical
                for name in ("sig", "rgbs", "dsig", "drgbs"):
                    assert np.array_equal(a[name][ia].view(np.uint32), b[name][ib].view(np.uint32)), (kw, name)
                if kw.get("overlap_optimizer") is False:
                    continue     # a sync step applies (and clears) its gradient inside the replay
                # the gradient: two atomic orders of the same terms
                e = np.abs(a["flat_grad"] - b["flat_grad"]).max() / np.abs(a["flat_grad"]).max()
                assert e <= 1e-5, (kw, e)
        # the applied updates: Adam's first step is lr * sign(g), so elements whose gradient changed sign between two
        # summation orders may differ by 2 lr; they must be a tiny share of the parameters
        far = ~np.isclose(gfin["flat_param"], ofin["flat_param"], rtol=1e-5, atol=1e-6)
        assert far.mean() < 1e-4, (kw, float(far.mean()))
        assert abs(gfin["losses"][1] - ofin["losses"][1]) <= 1e-4 * gfin["losses"][1]


# Graph step vs module path, flat gradient relative to its max.  Measured on an H100 over the three cases below: max
# 2.4e-7 .. 2.9e-7, p99.9 1.2e-8 .. 4.8e-8.
MODULE_MAX = 2e-6
MODULE_P999 = 3e-7


@pytest.mark.parametrize("w_d,reg", [(0.0, False), (1e-2, False), (0.0, True)])
def test_svox_graph_step_equals_module_path(monkeypatch, w_d, reg):
    from modules.distortion import distortion_loss
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    o, d, gt, noise = _batch(0)
    m1, t1, _ = _build(voxel_reg=REG if reg else None)
    monkeypatch.setattr(torch, "rand_like", lambda t, **k: noise.clone())
    extra = (lambda res: w_d * distortion_loss(res).mean()) if w_d > 0 else None
    loss1, _ = t1.forward_backward(o, d, gt, extra_loss=extra)
    monkeypatch.undo()
    torch.cuda.synchronize()
    g1 = t1.flat_grad.detach().cpu().numpy().copy()
    t1.optimizer_step()
    p1 = t1.flat_param.detach().cpu().numpy().copy()
    del t1, m1
    m2, t2, bits = _build(voxel_reg=REG if reg else None)
    fs = StaticTrainStep(t2, N_RAYS, samples_per_ray_capacity=CFG["spr"], T_threshold=THR, use_graph=True,
                         overlap_optimizer=True, distortion_loss_w=w_d)
    loss2 = float(fs.step(o, d, gt, noise=noise))
    snap = _snap(fs, bits)
    fs.flush()
    torch.cuda.synchronize()
    p2 = t2.flat_param.detach().cpu().numpy().copy()
    loss1 = float(loss1.detach())
    assert abs(loss1 - loss2) <= 2e-3 * loss1, (loss1, loss2)
    g2 = snap["flat_grad"]
    # both paths composite the fields' fp32 outputs in fp32; they differ in the summation order of the compositing and
    # of the atomics, so the bound is a few times what was measured, not the hash model's fp16 module-path bound
    e = np.abs(g2 - g1)
    scale = np.abs(g1).max()
    st = dict(max=float(e.max() / scale), p999=float(np.percentile(e[g1 != 0], 99.9) / scale))
    G._report(f"svox graph step vs module path, w_d={w_d} reg={reg}", st)
    assert st["max"] <= MODULE_MAX and st["p999"] <= MODULE_P999, st
    # after the update: equal within test_trainer_step_equals_torch_adam's bound wherever the two gradients agree in
    # sign (Adam's first step is lr * sign(g)); where they do not, the gradient is inside the bound above
    same = np.sign(g1) == np.sign(g2)
    assert np.allclose(p2[same], p1[same], rtol=2e-6, atol=1e-7)
    assert (np.abs(g1[~same]) <= MODULE_MAX * scale).all() and (~same).mean() < 1e-3


def _region_run(lat, n_steps=50):
    from datasets.synthetic import SyntheticLego
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, _ = _build(lat, voxel_reg=REG, den_range=(-1.0, 20.0), bits="full")
    block = m._reg_block
    keep_sh, keep_den = m.sh_fields.detach().clone(), m.density_fields.detach().clone()
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=512, T_threshold=THR, overlap_optimizer=True)
    ds = SyntheticLego(n_images=6, img_wh=(64, 64), focal=88.9, batch_size=N_RAYS, seed=2).to(DEV)
    ds.build_image_bank()
    fs.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=1234)
    dropped = torch.zeros((), device=DEV, dtype=torch.int64)
    for _ in range(n_steps):
        fs.step_sampled()
        dropped += fs.counter[1]
    fs.flush()
    torch.cuda.synchronize()
    out = torch.ones(keep_den.shape[:3], dtype=torch.bool, device=DEV)
    RR.block_of(out, block).fill_(False)
    (_, _, m_sh, v_sh), (_, _, m_den, v_den) = tr.voxel_fields()
    assert torch.equal(I32(m.sh_fields.detach())[out], I32(keep_sh)[out])
    assert torch.equal(I32(m.density_fields.detach())[out], I32(keep_den)[out])
    for t in (m_sh, v_sh, m_den, v_den):
        assert not bool(t[out].any())
    assert not bool(tr.flat_grad.any())
    assert not torch.equal(RR.block_of(m.sh_fields.detach(), block), RR.block_of(keep_sh, block))
    assert int(I32(fs.hyper[3:])) == n_steps and int(tr.found_inf) == 0
    print(f"\n[svox region] lattice {lat} B {block}: {n_steps} steps, {int(dropped)} rays cut short in all")
    return block


def test_svox_region_invariant_at_the_shipped_lattice():
    assert _region_run(dict(grid_size=256, grid_radius=0.0125, sh_degree=2)) == (86, 86, 86, 170, 170, 170)


def test_svox_region_invariant_with_b_clamped_to_the_lattice():
    """B clamped to the lattice is the whole grid here, so the outside-B half of the invariant is empty (it is exercised
    at the shipped lattice above).  What this case covers: samples whose corners reach the lattice's faces, the block
    pass over the whole grid and a zero flat_grad after the flush."""
    assert _region_run(dict(grid_size=83, grid_radius=0.0125, sh_degree=1)) == (0, 0, 0, 83, 83, 83)


# ---- 6. failure paths ---------------------------------------------------------------------------------------------
def test_svox_nan_at_b_far_corner_skips_the_step():
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, _ = _build(voxel_reg=(1.0, 0.0, 0.0))
    b = m._reg_block
    with torch.no_grad():
        m.density_fields[b[3] - 1, b[4] - 1, b[5] - 1, 0] = math.nan
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=CFG["spr"], T_threshold=THR)
    keep = [t.clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq)]
    fs.step(*_batch(0))
    torch.cuda.synchronize()
    for t, k in zip((tr.flat_param, tr.exp_avg, tr.exp_avg_sq), keep):
        assert torch.equal(I32(t), I32(k))
    assert int(I32(fs.hyper[3:])) == 0 and float(fs.scale_state[0]) == 2.0 ** 18
    assert int(tr.found_inf) == 1                # (cleared by the next step's reset)
    assert not bool(RR.block_of(tr.voxel_fields()[1][1], b).any())


def test_svox_poisoned_targets_skip_and_overflow_is_counted():
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    m, tr, bits = _build()
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=CFG["spr"], T_threshold=THR, overlap_optimizer=True)
    o, d, gt, noise = _batch(0)
    fs.step(o, d, gt, noise)
    fs.flush()
    keep = [t.clone() for t in (tr.flat_param, tr.exp_avg, tr.exp_avg_sq)]
    bad = gt.clone()
    bad[::97] = math.nan
    fs.step(o, d, bad, noise)
    fs.flush()
    torch.cuda.synchronize()
    for t, k in zip((tr.flat_param, tr.exp_avg, tr.exp_avg_sq), keep):
        assert torch.equal(t, k)
    assert int(I32(fs.hyper[3:])) == 1 and float(fs.scale_state[0]) == 2.0 ** 18
    assert not bool(tr.flat_grad.any())
    # capacity: far fewer rows than the rays march; the cut rays are counted and the step stays valid
    from oracle import oracle as O
    o_, d_, gt_, noise_ = _batch(1, dev=False)
    S_all = O.raymarching_train(o_, d_, O.ray_aabb_intersect(o_, d_, 0.5), bits, noise_, 1, 0.5, 0.0, 128, 1024)[5]
    m, tr, bits = _build()
    fs = StaticTrainStep(tr, N_RAYS, samples_per_ray_capacity=(S_all - 3000) // N_RAYS, T_threshold=THR,
                         overlap_optimizer=True)
    fs.step(*_batch(1))
    snap = _snap(fs, bits)
    fs.flush()
    mm = G.check_march(snap, CFG)
    assert snap["counter"][0] == S_all > fs.cap and mm["cut"] >= 1 and snap["counter"][1] == mm["cut"], mm
    assert snap["found_inf"] == 0 and np.isfinite(snap["flat_param"]).all()
    assert int(I32(fs.hyper[3:])) == 1
    check_voxel_stages(snap, _lay())


def test_svox_refusals_and_other_models_kernel_counts():
    from modules.networks import NGP
    from taichi_nerfs_b200._lib import NgpError
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    m, tr, _ = _build(dict(grid_size=16, grid_radius=0.0625, sh_degree=0))
    tr.world_size = 2
    with pytest.raises(NgpError):
        StaticTrainStep(tr, 256, samples_per_ray_capacity=64)
    counts = {}
    for name, kw in (("hash", dict(half_opt=True)), ("triplane", dict(half_opt=False, pos_encoder_type="triplane"))):
        mm = NGP(scale=0.5, max_res=1024, **kw).cuda()
        t = NGPTrainer(mm)
        fs = StaticTrainStep(t, 8192, overlap_optimizer=True)       # the configuration of the §6b table
        counts[name] = fs.kernels_per_replay
        del fs, t, mm
    assert counts == dict(hash=12, triplane=11), counts     # + the sampler: 13 and 12 (DESIGN.md §6b table)


# ---- 7. end to end --------------------------------------------------------------------------------------------------
def _train_graph(reg, steps=1000):
    from datasets.ray_utils import get_rays
    from modules.rendering import MAX_SAMPLES, render
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    from test_gpu_e2e import _small_dataset
    torch.manual_seed(23)
    ds = _small_dataset(root_dir='', split='train', downsample=1.0, seed=23, scene='analytic').to(DEV)
    ds.batch_size = 4096
    ds.build_image_bank()
    test = _small_dataset(root_dir='', split='test', downsample=1.0, n_images=4, scene='analytic').to(DEV)
    m = VoxelGrid().to(DEV)
    m.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    tr = NGPTrainer(m, lr=1e-2, max_steps=steps, voxel_reg=reg)
    fs = StaticTrainStep(tr, 4096, samples_per_ray_capacity=1024, overlap_optimizer=True)
    fs.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=23)
    cut = torch.zeros((), device=DEV, dtype=torch.int64)     # rays cut short, summed over every step on the device
    rows = torch.zeros((), device=DEV, dtype=torch.int32)
    for step in range(steps):
        if step % 16 == 0:
            fs.flush()
            with torch.autocast(device_type='cuda', dtype=torch.float16):
                m.update_density_grid(0.01 * MAX_SAMPLES / 3 ** 0.5, warmup=step < 256)
        fs.step_sampled()
        cut += fs.counter[1]
        rows = torch.maximum(rows, fs.counter[0])
    cut, rows = int(cut), int(rows)
    fs.flush()
    m.eval()
    psnrs = []
    with torch.no_grad():
        for i in range(len(test)):
            td = test[i]
            with torch.autocast(device_type='cuda', dtype=torch.float16):
                o, d = get_rays(test.directions, td['pose'])
                res = render(m, o, d, test_time=True)
            mse = torch.nn.functional.mse_loss(res['rgb'].float(), td['rgb'])
            psnrs.append(float(-10 * torch.log10(mse)))
    print(f"\n[svox graph e2e reg={reg}] psnr {psnrs}, rays cut over all steps {cut}, most rows {rows} "
          f"of {fs.cap}")
    return psnrs, cut


# Measured once on an H100 80GB HBM3 at a 700 W power limit, 1000 graph steps, dB per held-out view (no ray cut).  The gates are the module path's
# (test_gpu_voxel_grid.PSNR_GATE, test_gpu_voxel_reg.PSNR_GATE).
PSNR_MEASURED = {"plain": [18.42, 19.99, 20.75, 20.01], "reg": [18.63, 20.16, 20.94, 20.31]}


@pytest.mark.parametrize("reg", [None, REG])
def test_svox_graph_training_reaches_the_module_path_gate(reg):
    psnrs, cut = _train_graph(reg)
    assert cut == 0
    assert min(psnrs) > (16.6 if reg else 16.4), psnrs
