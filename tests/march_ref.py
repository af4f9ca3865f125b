"""Independent restatement of the reference's occupancy-grid ray march, and fp64 checks of emitted samples.

The marcher (``csrc/march.cu``) is held bit-exact to the C oracle (``oracle/ngp_oracle.c``), which is our own port of
the reference, so a mistake made in both would pass every parity test.  This module restates the same march a second
time, straight from the reference and in numpy fp32 (every operation rounded to fp32 on its own, no fused multiply-add),
vectorised over rays with one loop over steps:

* ``aabb``          -- ``modules/intersection.py:8-37``
* ``march_train``   -- ``modules/ray_march.py:27-74`` (the count loop; the write loop at :83-123 visits the same
                        positions) with the helpers of ``modules/utils.py:54-117``
* ``march_test``    -- ``modules/ray_march.py:197-268``

Quirks of the reference that are kept, because they decide which cell a sample is looked up in:

* ``frexp_bit(0) = 0`` (utils.py:62-63), so a sample exactly at the origin has ``mip_from_pos = 1``, not 0.
* ``frexp_bit`` returns ``ceil(log2 x)``: an exact power of two keeps its exponent (utils.py:70-73), unlike C's
  ``frexp``.
* The exit of an empty cell is computed from the clamped but un-floored grid coordinate (ray_march.py:68-69), so
  along an axis with ``d < 0`` the "exit" is the sample itself and the loop advances by one step.
* ``sign(0) = 0`` (``ti.math.sign``, ray_march.py:68): an axis-parallel component contributes ``nxyz + 0.5``.
* The grid coordinate is clamped to ``[0, G - 1]`` before the cast to an integer cell (ray_march.py:54-60).
* The noise jitter of the start applies only when ``t1 >= 0`` (ray_march.py:38-40).
* The test march requires strict ``0 < t`` (ray_march.py:230); the training march ``0 <= t`` (:45).

The reference never ends a ray whose ``t + dt`` stops increasing (a far hit at ``+inf`` from a zero or NaN direction,
or one so far that fp32 ``t + dt`` rounds back to ``t``).  The restatement follows it, so it raises
``StepBudgetExceeded`` instead of looping past ``budget`` steps; that is how it reports those rays.

``check_samples`` holds for the output of any correct marcher, whatever its arithmetic order: each sample in
``[t1, t2)``, strictly increasing per ray, on its ray within fp32 rounding, with the reference's step size, and in an
occupied cell of the cascade the reference picks (computed in fp64).  A mistake the oracle and the kernel share fails
it.

``fault=`` plants one deliberate mistake in the restatement (``FAULTS``), so the tests can show that the checks reject
each of them.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
NEAR_DISTANCE = f32(0.01)                                      # utils.py:13
SQRT3 = 1.7320508075688772
SQRT3_MAX_SAMPLES = f32(SQRT3 / 1024)                          # utils.py:15
SQRT3_2 = f32(SQRT3 * 2)                                       # utils.py:16

FAULTS = ("mip_bound_x2", "morton_swap_xy", "clamp_at_G", "frexp_std", "dt_max_scale_over_G", "no_cascade_offset")


class StepBudgetExceeded(RuntimeError):
    """Some ray did not end within the step budget (the reference would loop forever on it)."""


def aabb(rays_o, rays_d, scale):
    """hits_t [n, 2] of intersection.py:8-37 (fp32, ``fmin``/``fmax`` drop NaN like the device min/max)."""
    o, d = np.asarray(rays_o, f32), np.asarray(rays_d, f32)
    s = f32(scale)
    half = f32((s - (-s)) / f32(2))                             # :15-17
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = f32(1) / d                                        # :24
        tmin = (f32(0) - half - o) * inv                        # :26
        tmax = (f32(0) + half - o) * inv                        # :27
        lo, hi = np.fmin(tmin, tmax), np.fmax(tmin, tmax)       # :29-30
    t1 = np.fmax(np.fmax(lo[:, 0], lo[:, 1]), lo[:, 2])         # :31
    t2 = np.fmin(np.fmin(hi[:, 0], hi[:, 1]), hi[:, 2])         # :32
    hit = t2 > 0                                                # :34
    out = np.full((o.shape[0], 2), -1.0, f32)
    out[hit, 0] = np.fmax(t1[hit], NEAR_DISTANCE)
    out[hit, 1] = t2[hit]
    return out


def _frexp_bit(x, fault=None):
    """utils.py:60-75 on an fp32 array: ceil(log2 |x|) for x != 0, and 0 for x == 0."""
    x = np.asarray(x, f32)
    if fault == "frexp_std":
        return np.frexp(x)[1].astype(np.int64)
    bits = x.view(np.uint32)
    e = ((bits & np.uint32(0x7F800000)) >> np.uint32(23)).astype(np.int64) - 127
    frac = ((bits & np.uint32(0x7FFFFF)) | np.uint32(0x3F800000)).view(f32)
    e = e - (frac < f32(0.5)) + (frac > f32(1.0))
    return np.where(x != 0, e, 0)


def _expand_bits(v):                                            # utils.py:95-100 (uint32, wrapping products)
    v = np.asarray(v, np.uint32)
    v = (v * np.uint32(0x00010001)) & np.uint32(0xFF0000FF)
    v = (v * np.uint32(0x00000101)) & np.uint32(0x0F00F00F)
    v = (v * np.uint32(0x00000011)) & np.uint32(0xC30C30C3)
    v = (v * np.uint32(0x00000005)) & np.uint32(0x49249249)
    return v


def morton3d(u, fault=None):                                    # utils.py:103-107
    x, y, z = u[:, 0], u[:, 1], u[:, 2]
    if fault == "morton_swap_xy":
        x, y = y, x
    return _expand_bits(x) | (_expand_bits(y) << np.uint32(1)) | (_expand_bits(z) << np.uint32(2))


class _Cfg:
    def __init__(self, cascades, scale, esf, G, fault):
        self.C, self.G, self.fault = int(cascades), int(G), fault
        self.scale, self.esf, self.gsf = f32(scale), f32(esf), f32(G)
        self.gs_inv = f32(f32(1) / self.gsf)                    # ray_march.py:36
        self.gs3 = self.G ** 3
        top = self.scale if fault == "dt_max_scale_over_G" else f32(SQRT3_2 * self.scale)
        self.dt_max = f32(top / self.gsf)                       # utils.py:56-57: SQRT3_2 * scale / grid_size

    def calc_dt(self, t):                                       # utils.py:54-57: clamp(t * esf, lo, hi)
        return np.fmin(np.fmax(t * self.esf, SQRT3_MAX_SAMPLES), self.dt_max)


def _lookup(cfg, bits, xyz, dt):
    """Cascade, clamped grid coordinate and occupancy of fp32 positions (ray_march.py:46-61)."""
    F = cfg.fault
    mx = np.fmax(np.fmax(np.abs(xyz[:, 0]), np.abs(xyz[:, 1])), np.abs(xyz[:, 2]))
    m_pos = np.clip(_frexp_bit(mx, F) + 1, 0, cfg.C - 1)        # utils.py:78-84
    m_dt = np.clip(_frexp_bit(dt * cfg.gsf, F), 0, cfg.C - 1)   # utils.py:87-92
    mip = np.maximum(m_pos, m_dt)
    p2 = (mip if F == "mip_bound_x2" else mip - 1).astype(np.float64)
    mip_bound = np.fmin(np.exp2(p2).astype(f32), cfg.scale)     # ray_march.py:51: min(pow(2, mip - 1), scale)
    inv = (f32(1) / mip_bound)[:, None]
    v = f32(0.5) * (xyz * inv + f32(1)) * cfg.gsf               # :54-58, left to right
    top = cfg.gsf if F == "clamp_at_G" else f32(cfg.gsf - f32(1))
    nxyz = np.fmin(np.fmax(v, f32(0)), top)
    cell = morton3d(nxyz.astype(np.uint32), F).astype(np.int64)  # :60, the cast after the clamp
    idx = cell if F == "no_cascade_offset" else mip * cfg.gs3 + cell
    byte = bits[(idx >> 3) % bits.size]                         # (the modulo only keeps a planted fault in range)
    occ = ((byte >> (idx & 7)) & 1).astype(bool)                # :61
    return mip_bound, nxyz, occ


def _march(o, d, t_start, t2, bits, cfg, max_samples, strict, budget):
    """The loop of ray_march.py:45-74 / :230-266 for all rays at once.  Returns per-ray sample lists as flat arrays in
    ray order plus the per-ray count and the position after the last sample (the test march's resume point)."""
    n = o.shape[0]
    with np.errstate(divide="ignore"):
        d_inv = f32(1) / d                                      # ray_march.py:31
    sgn = np.sign(d).astype(f32)
    t = t_start.astype(f32).copy()
    count = np.zeros(n, np.int64)
    resume = np.full(n, np.nan, f32)
    skipping = np.zeros(n, bool)
    t_target = np.zeros(n, f32)
    rec = []
    steps = 0
    with np.errstate(invalid="ignore", over="ignore"):
        while True:
            go = (0 < t) if strict else (0 <= t)
            visit = ~skipping & go & (t < t2) & (count < max_samples)
            if not (visit.any() or skipping.any()):
                break
            steps += 1
            if steps > budget:
                bad = np.nonzero(visit | skipping)[0]
                raise StepBudgetExceeded(f"{bad.size} rays still marching after {budget} steps, e.g. ray {bad[0]} "
                                         f"at t = {t[bad[0]]!r}")
            # inner skip loop of an empty cell, one step per pass: while t < t_target: t += calc_dt(t) (:73-74)
            s = np.nonzero(skipping)[0]
            if s.size:
                ts = t[s] + cfg.calc_dt(t[s])
                t[s] = ts
                skipping[s] = ts < t_target[s]
            r = np.nonzero(visit)[0]
            if r.size == 0:
                continue
            tr = t[r]
            xyz = o[r] + tr[:, None] * d[r]                     # :46
            dt = cfg.calc_dt(tr)                                # :47
            mip_bound, nxyz, occ = _lookup(cfg, bits, xyz, dt)
            e = r[occ]
            if e.size:
                rec.append((e, tr[occ], dt[occ], xyz[occ]))
                t[e] = tr[occ] + dt[occ]                        # :64
                count[e] += 1
                resume[e] = t[e]                                # :257
            m = ~occ
            q = r[m]
            if q.size:                                          # :68-74
                a = (((nxyz[m] + f32(0.5) + f32(0.5) * sgn[q]) * cfg.gs_inv * f32(2) - f32(1))
                     * mip_bound[m][:, None] - xyz[m]) * d_inv[q]
                tmin = np.fmin(np.fmin(a[:, 0], a[:, 1]), a[:, 2])
                t_target[q] = tr[m] + np.fmax(f32(0), tmin)
                t[q] = tr[m] + dt[m]
                skipping[q] = t[q] < t_target[q]
    if rec:
        ray = np.concatenate([x[0] for x in rec])
        order = np.argsort(ray, kind="stable")                  # a ray's samples were recorded in step order
        ray = ray[order]
        ts, dts = (np.concatenate([x[i] for x in rec])[order] for i in (1, 2))
        xyzs = np.concatenate([x[3] for x in rec])[order]
    else:
        ray, ts, dts, xyzs = np.zeros(0, np.int64), np.zeros(0, f32), np.zeros(0, f32), np.zeros((0, 3), f32)
    return ray, ts, dts, xyzs, count, resume


def march_train(rays_o, rays_d, hits_t, bits, cascades, scale, esf, G, max_samples, noise=None, fault=None,
                budget=1 << 15):
    """ray_march.py:27-74 (+ the write loop's identical visits, :83-123).  Returns (counts [n], ray [S], ts [S],
    deltas [S], xyzs [S, 3]) with the samples in ray order, like the oracle's and the module's layout."""
    o, d, h = (np.ascontiguousarray(a, f32) for a in (rays_o, rays_d, hits_t))
    cfg = _Cfg(cascades, scale, esf, G, fault)
    t1 = h[:, 0].copy()
    if noise is not None:
        j = t1 >= 0                                             # :38-40
        with np.errstate(invalid="ignore"):                     # t1 = +inf (a tangent ray on a - face): inf * 0
            t1[j] = t1[j] + cfg.calc_dt(t1[j]) * np.asarray(noise, f32)[j]
    ray, ts, dts, xyzs, count, _ = _march(o, d, t1, h[:, 1], np.asarray(bits, np.uint8), cfg, max_samples, False,
                                          budget)
    return count, ray, ts, dts, xyzs


def march_test(rays_o, rays_d, hits_t, alive, bits, cascades, scale, esf, G, max_samples, fault=None,
               budget=1 << 15):
    """ray_march.py:197-268 for the rays ``alive``.  Returns (counts [A], ts [A, max_samples], deltas
    [A, max_samples], new hits_t) -- unused slots 0, hits_t[r, 0] moved past the last sample of each ray with one."""
    o, d, h = (np.ascontiguousarray(a, f32) for a in (rays_o, rays_d, hits_t))
    alive = np.asarray(alive, np.int64)
    cfg = _Cfg(cascades, scale, esf, G, fault)
    ray, ts, dts, _, count, resume = _march(o[alive], d[alive], h[alive, 0], h[alive, 1], np.asarray(bits, np.uint8),
                                            cfg, max_samples, True, budget)
    A = alive.size
    T, D = np.zeros((A, max_samples), f32), np.zeros((A, max_samples), f32)
    slot = np.arange(ray.size) - np.repeat(np.cumsum(count) - count, count)
    T[ray, slot], D[ray, slot] = ts, dts
    h_new = h.copy()
    moved = count > 0
    h_new[alive[moved], 0] = resume[moved]
    return count, T, D, h_new


# ---- fp64 checks of emitted samples ----------------------------------------------------------------------------------
U = 2.0 ** -24                                                  # unit roundoff of fp32


def _fail(what, i, **kv):
    extra = ", ".join(f"{k}={v!r}" for k, v in kv.items())
    raise AssertionError(f"{what}: sample {i} ({extra})")


def check_samples(rays_o, rays_d, hits_t, ray, ts, deltas, xyzs, bits, cascades, scale, esf, G=128):
    """Properties every correct march output has, checked in fp64 against the reference's definitions.

    ``ray`` gives each sample's ray (samples of a ray in emission order, rays in any order); ``hits_t`` the interval
    the march was given.  Raises AssertionError naming the first sample that breaks one of:
      * ``t1 <= t < t2`` and t strictly increasing along each ray;
      * ``xyz`` within fp32 rounding of fp64 ``o + t d``: ``|xyz - (o + t d)| <= u (|t d| + |xyz|)``;
      * ``dt = clamp(t * esf, sqrt3/1024, 2 sqrt3 scale / G)`` within the rounding of its three fp32 constants;
      * the cascade is the smallest one that contains the point (``2^(m-1) >= max|x|``) and whose cells are at least
        dt (``2^m / G >= dt``), capped at the top one.  The one exception is ``max|x| = 0``, where the reference's
        ``frexp_bit(0) = 0`` gives cascade 1;
      * the fp64 cell of xyz in that cascade is set in the bitfield.  Where a coordinate lies within the fp32 window
        of a cell face, either neighbour is accepted.
    """
    o = np.asarray(rays_o, np.float64)
    d = np.asarray(rays_d, np.float64)
    h = np.asarray(hits_t, np.float64)
    ray = np.asarray(ray, np.int64)
    t = np.asarray(ts, np.float32).astype(np.float64)
    dt = np.asarray(deltas, np.float32).astype(np.float64)
    x = np.asarray(xyzs, np.float32).astype(np.float64).reshape(-1, 3)
    n = t.size
    if n == 0:
        return
    scale = float(np.float32(scale))
    C = int(cascades)

    bad = np.nonzero(~((h[ray, 0] <= t) & (t < h[ray, 1])))[0]
    if bad.size:
        i = bad[0]
        _fail("t outside [t1, t2)", i, ray=int(ray[i]), t=t[i], hits=tuple(h[ray[i]]))
    same = ray[1:] == ray[:-1]
    bad = np.nonzero(same & ~(t[1:] > t[:-1]))[0]
    if bad.size:
        i = bad[0] + 1
        _fail("t not strictly increasing along the ray", i, ray=int(ray[i]), t=t[i], previous=t[i - 1])

    td = t[:, None] * d[ray]                                    # exact: fp32 x fp32 fits fp64
    err = np.abs(x - (o[ray] + td))
    bad = np.nonzero((err > U * (np.abs(td) + np.abs(x)) * (1 + 4 * U) + 2.0 ** -149).any(1))[0]
    if bad.size:
        i = bad[0]
        _fail("xyz off the ray", i, ray=int(ray[i]), t=t[i], xyz=tuple(x[i]), exact=tuple(o[ray[i]] + td[i]))

    want = np.clip(t * float(esf), SQRT3 / 1024, 2 * SQRT3 * scale / G)
    bad = np.nonzero(np.abs(dt - want) > 3 * U * want)[0]
    if bad.size:
        i = bad[0]
        _fail("dt is not clamp(t * esf, sqrt3/1024, 2 sqrt3 scale / G)", i, t=t[i], dt=dt[i], want=want[i])

    mx = np.abs(x).max(1)
    m = np.arange(C)
    fits_pos = np.exp2(m - 1.0)[None, :] >= mx[:, None]
    fits_dt = (np.exp2(m * 1.0) / G)[None, :] >= dt[:, None]
    ok = fits_pos & fits_dt
    mip = np.where(ok.any(1), ok.argmax(1), C - 1)
    at_origin = mx == 0
    mip[at_origin] = np.maximum(mip[at_origin], min(1, C - 1))  # frexp_bit(0) = 0 -> mip_from_pos = 1

    mb = np.minimum(np.exp2(mip - 1.0), scale)
    v = 0.5 * (x / mb[:, None] + 1.0) * G                       # fp64 grid coordinate
    w = 2.0 ** -21 * G                                          # fp32 window of a face, in grid units (8 fp32 ulps)
    lo = np.clip(np.floor(v - w), 0, G - 1).astype(np.int64)
    hi = np.clip(np.floor(v + w), 0, G - 1).astype(np.int64)
    bitv = np.unpackbits(np.asarray(bits, np.uint8), bitorder="little")
    base = mip * G ** 3
    occupied = np.zeros(n, bool)
    for cx in (lo[:, 0], hi[:, 0]):                             # every neighbour a face window allows
        for cy in (lo[:, 1], hi[:, 1]):
            for cz in (lo[:, 2], hi[:, 2]):
                cell = morton3d(np.stack([cx, cy, cz], 1).astype(np.uint32)).astype(np.int64)
                occupied |= bitv[base + cell].astype(bool)
    bad = np.nonzero(~occupied)[0]
    if bad.size:
        i = bad[0]
        _fail("sample in an empty cell (fp64 cell of the reference's cascade)", i, ray=int(ray[i]), t=t[i],
              xyz=tuple(x[i]), cascade=int(mip[i]), coord=tuple(v[i]))


# ---- rays at the edges of the march ----------------------------------------------------------------------------------
def binade_start(B, lane, dt):
    """fp32 start t0 of the constant-dt chain t_{k+1} = t_k + dt whose step from position ``lane`` to ``lane + 1``
    crosses the binade boundary B (t_lane < B <= t_lane+1)."""
    B, dt = f32(B), f32(dt)
    lo, hi = np.float64(B) - (lane + 2) * float(dt), np.float64(B) - (lane - 1) * float(dt)
    for _ in range(80):                                         # the crossing index falls as t0 grows: bisect
        g = f32((lo + hi) / 2)
        chain = [g]
        for _ in range(lane + 1):
            chain.append(f32(chain[-1] + dt))
        if chain[lane] >= B:
            hi = float(g)
        elif chain[lane + 1] < B:
            lo = float(g)
        else:
            return g
    raise AssertionError("no start found")


def edge_rays(scale, G=128, seed=0):
    """(rays_o, rays_d, hits_t, names): rays at the edges of the march, all of which end, with the interval each one
    is marched over (from ``aabb``, or chosen by the caller where the start matters).  ``names[i]`` says what ray i
    is.  Inside-the-box starts use scale 0.5 geometry, so every configuration with scale >= 0.5 holds them."""
    rng = np.random.default_rng(seed)
    s = f32(scale)
    O, D, H, names = [], [], [], []

    def add(o, d, name, hits=None):
        o, d = np.asarray(o, f32).reshape(3), np.asarray(d, f32).reshape(3)
        O.append(o)
        D.append(d)
        H.append(aabb(o[None], d[None], s)[0] if hits is None else np.asarray(hits, f32))
        names.append(name)

    # axis-parallel directions, with +0 and -0 components, from inside the box and from outside it
    for ax in range(3):
        for sg in (1.0, -1.0):
            for zero in (0.0, -0.0):
                d = np.full(3, zero)
                d[ax] = sg
                for k in range(2):
                    o = rng.uniform(-0.45, 0.45, 3)
                    add(o, d, f"axis{ax}{'+-'[sg < 0]}{'neg0' if str(zero)[0] == '-' else '0'}_in{k}")
                o = rng.uniform(-0.4, 0.4, 3)
                o[ax] = -sg * (float(s) + 0.3)
                add(o, d, f"axis{ax}{'+-'[sg < 0]}_out")
    for k in range(6):                                           # two live axes, one zero component
        d = rng.normal(size=3)
        d[k % 3] = -0.0 if k >= 3 else 0.0
        add(rng.uniform(-0.4, 0.4, 3), d / np.linalg.norm(d), f"plane_zero{k}")
    # origins on cell faces (cascade 0: faces every 1/G) and exactly on the AABB faces
    for k in range(12):
        o = (rng.integers(-G // 2 + 2, G // 2 - 2, 3) / G).astype(f32)
        d = rng.normal(size=3)
        add(o, d / np.linalg.norm(d), f"cell_face_origin{k}")
    for ax in range(3):
        for sg in (1.0, -1.0):
            o = rng.uniform(-0.4, 0.4, 3)
            o[ax] = sg * float(s)
            d_in = rng.normal(size=3)
            d_in[ax] = -sg * abs(d_in[ax]) - 0.2
            add(o, d_in / np.linalg.norm(d_in), f"aabb_face{ax}{'+-'[sg < 0]}_inward")
            d_t = rng.normal(size=3)
            d_t[ax] = 0.0                                       # tangent: marches along the face
            add(o, d_t / np.linalg.norm(d_t), f"aabb_face{ax}{'+-'[sg < 0]}_tangent")
    # positions with max|x| an exact power of two: a coordinate held at +-0.5, +-1, +-2 by a zero component, the others
    # small (the cascade of such a point is the one exactly as large; clamped to G - 1 at its + face)
    for a in (0.5, 1.0, 2.0):
        if a > s:
            continue
        for sg in (1.0, -1.0):
            o = np.array([sg * a, -0.35 * a, 0.1 * a])
            add(o, [0.0, 0.96, 0.28], f"pow2_face{a}{'+-'[sg < 0]}", hits=[0.01, 0.65 * a])
    # rays through the exact origin: o = -t0 d with exact products, started at t0 (the first sample is at 0, 0, 0)
    for k, (d, t0) in enumerate((([0.5, 0.25, -0.75], 0.5), ([-0.625, 0.5, 0.125], 0.25), ([0.0, -1.0, 0.0], 0.375))):
        d = np.asarray(d, f32)
        o = -f32(t0) * d
        add(o, d, f"through_origin{k}", hits=[t0, aabb(o[None], d[None], s)[0, 1]])
    # grazing rays: nearly parallel to a face, just inside it; and rays that clip a box edge
    for k, eps in enumerate((1e-7, 1e-5, 1e-3)):
        o = np.array([-float(s) - 0.2, float(s) - 1e-6, 0.1])
        add(o, [1.0, eps, 0.0], f"graze_face{k}")
    for k, off in enumerate((1e-6, 1e-4)):
        o = np.array([-float(s) - 0.1, float(s) + 0.1 - off, 0.0])
        add(o, np.array([1.0, -1.0, 0.0]) / np.sqrt(2), f"clip_edge{k}")
    # direction components at the `regular` threshold of the warp march: d < -1e-3 is the negative-axis test
    thr = f32(-1e-3)
    for k, c in enumerate((thr, np.nextafter(thr, f32(0)), np.nextafter(thr, f32(-1)))):
        o = rng.uniform(-0.3, 0.3, 3)
        add(o, [c, 0.6, 0.8], f"dir_minus1e-3_{k}")
        add(o, [c, c, -0.99], f"dir_minus1e-3_two_axes{k}")
    # constant-dt chains whose binade boundary B falls between position `lane` and `lane + 1` of a 32-position chunk
    dt = f32(SQRT3_MAX_SAMPLES)
    for B in (0.5, 1.0, 2.0):
        for lane in (0, 1, 15, 31, 32):
            t0 = binade_start(B, lane, dt)
            d = np.array([0.8, 0.36, -0.48], f32)
            o = (np.array([0.1, -0.2, 0.05]) - B * d.astype(np.float64)).astype(f32)
            add(o, d, f"binade{B}_lane{lane}", hits=[t0, aabb(o[None], d[None], s)[0, 1]])
    return np.stack(O), np.stack(D), np.stack(H).astype(f32), names


def degenerate_rays():
    """(rays_o, rays_d, names): rays the reference marches forever once given an interval [0.01, t2) with no finite t2
    (zero or NaN direction, NaN origin), or with a t2 so distant (direction 1e-30, t2 ~ 2e29) that fp32 t + dt stops
    increasing before it.  (Of the first three, the reference's own AABB test gives [0.01, +inf) to the zero direction;
    the NaN rays reach the march through a caller's interval.)"""
    nan = np.nan
    o = np.array([[0.1, 0.2, -0.1], [0.1, 0.2, -0.1], [nan, nan, nan], [0.1, 0.2, -0.1]], f32)
    d = np.array([[0.0, 0.0, 0.0], [nan, nan, nan], [0.6, 0.8, 0.0], [1e-30, 1e-30, 1e-30]], f32)
    return o, d, ["zero_direction", "nan_direction", "nan_origin", "direction_1e-30"]
