"""The F = 2 hash kernels' lane walk (hash_fwd_kernel, hash_bwd_kernel in taichi_nerfs_b200/csrc/hash.cu) on
constructed sample streams, against references that have no per-row state: the oracle's forward bit for bit, and the
fp64 scatter of tests/hash_ref.py within its any-order bound.

A lane walks 16 consecutive rows of one level and keeps state from row to row.  The forward re-gathers the 8 corners
only when the cell changes.  The backward carries the corners that two neighbouring cells share (cell_step,
shift_corners), flushes only the corners that leave, and sends a leaving x-pair in one 16-byte reduction.  Uniform
points almost never take the carry path, and straight rays never reverse, so the streams here script the path of
cells at one level at a time (level 0, a dense middle level, the first hashed level and the finest):

- every neighbour move d in {-1, 0, 1}^3 \\ {0}, each followed by its reverse, with runs of 1 to 5 rows per cell:
  the backward's carried and leaving masks for every move;
- oscillation A B A B, +-2 on one axis and a jump back to an earlier cell: a flush of all 8 corners inside a walk;
- rows whose dy is zero at the scripted level, inside a run and between two runs.  Rows zero at every level sit at
  NaN positions, so a walk that did not skip them would scatter NaN; rows zero at the scripted level only sit in
  another cell.  Other rows are zero at other levels only;
- each path at every offset 0-15 of a lane's 16-row chunk, placed so that runs cross the 512-row CTA boundaries;
- points exactly on cell faces, at x = 0 and x = 1 (where a dense level's corner index passes its size and wraps),
  and slightly outside the box: the grid coordinate past the resolution, and in fp32 negative.  In fp16 a negative
  grid coordinate casts to f16(2^32) = inf (the fp16 grid cast, hash_encoder_half.py:132), so the fp16 streams keep
  x >= 0.

A table of 1000 entries per level (see _layout) makes the hashed levels collide often: two corners of one cell, or a
carried and a leaving corner of one move, share an entry.  test_walk_streams_exercise_every_path counts every category in the
streams, and test_check_scatter_rejects_seeded_walk_faults shows that the backward's bound rejects a misplaced carried
corner, a dropped leaving corner and a swapped merged x-pair.

The same comparisons run at L in {1, 2, 3, 5, 8, 11, 16}, and at L = 16 with out / dL/dout one entry past a 16-byte
aligned allocation.  L % kVec != 0 (kVec = 2 for fp32, 4 for fp16: L = 3, 5, 11, and 2 in fp16) and the offset views
take the kernels' scalar staging and write-out branches.  Row counts n in {1, 15, 16, 17, 511, 512, 513, 1025} and the
whole stream; the device row count (_dyn); level ranges of ngp_hash_encode_bwd_levels, every [a, b) at L = 5 and
ranges whose ends are not multiples of kVec at L = 16.
"""
import ctypes as C
import functools
import itertools
from typing import NamedTuple

import numpy as np
import pytest
import torch

from taichi_nerfs_b200.layout import make_hash_layout

from hash_ref import (PAD, _check_scatter, _level_ranges, _level_slice, corner_entries, grid_cell, n_dev_cases,
                      np_hash_bwd_f64, rows_of)

DEV = "cuda"
F32, F16 = 0, 1
CHUNK, CTA = 16, 512
LEVEL_COUNTS = (1, 2, 3, 5, 8, 11, 16)
N_ROWS = (1, 15, 16, 17, 511, 512, 513, 1025)
MOVES = {d for d in itertools.product((-1, 0, 1), repeat=3) if any(d)}
SENTINEL = -7.0


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def N(t):
    return t.detach().cpu().numpy()


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def ST():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def chk(rc):
    from taichi_nerfs_b200 import _lib
    _lib.check(rc)


def i32(v):
    return torch.tensor([v], device=DEV, dtype=torch.int32)


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


# ---- streams ----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _layout(L):
    """1000 entries per level, resolutions 4 to 256: dense levels up to resolution 10, hashed ones above.  1000 is not
    a power of two, so the hashed levels take the kernels' modulo (h % size, not h & mask), and their entries collide
    as a random map's would: ~1-3 % of cells have two corners on one entry.  With 2^10 entries the xor hash of
    neighbouring coordinates almost never collides (no cell at all at resolution 13)."""
    return make_hash_layout(1000, L, 4, 256, 2)


def _scripted_levels(lay):
    """Level 0, a dense middle level, the first hashed level and the finest (fewer where they coincide)."""
    fh, L = lay.begin_fast_hash_level, lay.levels
    return sorted({0, fh // 2, min(fh, L - 1), L - 1})


def _f32_pos(x, s):
    """fp32(fp32(x * scale) + 0.5): the forward's grid position."""
    return (np.float32(x) * np.float32(s)).astype(np.float32) + np.float32(0.5)


def _face(s, g):
    """An fp32 x whose grid position is exactly g (fraction 0: on the face between cells g - 1 and g), or None."""
    x0 = np.float32((g - 0.5) / float(s))
    up = down = x0
    for _ in range(64):
        for c in (up, down):
            if _f32_pos(c, s) == np.float32(g):
                return c
        up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(-np.inf))
    return None


def _cell_points(lay, lvl, cells, rng, faces, nonneg):
    """fp32 points of the given cells at level lvl, fractions in [0.05, 0.95] ([0.5, 0.95] on an axis at g = 0 when
    nonneg, so that x >= 0); the rows in `faces` are moved onto the lower face of their cell on one axis."""
    s = lay.scales[lvl]
    cells = np.asarray(cells, np.int64).reshape(-1, 3)
    f = rng.uniform(0.05, 0.95, cells.shape)
    if nonneg:
        f = np.where(cells == 0, rng.uniform(0.5, 0.95, cells.shape), f)
    x = ((cells + f - 0.5) / s).astype(np.float32)
    for i in np.flatnonzero(faces):
        axes = [d for d in range(3) if not (nonneg and cells[i, d] <= 0)]     # the face of g = 0 lies at x < 0
        d = int(rng.choice(axes))
        xf = _face(s, cells[i, d])
        if xf is not None:
            x[i, d] = xf
    g, _ = grid_cell(x, lay, lvl, False)
    assert np.array_equal(g.view(np.int32), cells), "a scripted point left its cell"
    return x


class _Rows:
    """Rows under construction: position, the levels whose dy is zero, and a run id (the visit of a scripted cell the
    row belongs to, -1 for skipped and filler rows)."""

    def __init__(self, L):
        self.L, self.x, self.zero, self.run = L, [], [], []

    def add(self, x, zero, run):
        x = np.asarray(x, np.float32).reshape(-1, 3)
        self.x.append(x)
        self.zero.append(np.broadcast_to(np.asarray(zero, bool), (len(x), self.L)))
        self.run.append(np.broadcast_to(run, len(x)))

    def arrays(self):
        return np.concatenate(self.x), np.concatenate(self.zero), np.concatenate(self.run)


def _other_zero(rng, L, lvl, k=1):
    """Rows live at lvl with dy zero at some other levels (one level in twenty)."""
    z = rng.random((k, L)) < 0.05
    z[:, lvl] = False
    return z


def _carry_collides(lay, lvl, A):
    """Whether a move between cell A and one of its neighbours carries a corner whose entry is also the entry of a
    corner that leaves."""
    around = {d: i for i, d in enumerate(itertools.product((-1, 0, 1), repeat=3))}
    g = (A + np.array(list(around), np.int64)).astype(np.uint32)
    ent = np.stack([corner_entries(lay, lvl, g, c) for c in range(8)], 1)
    for d in MOVES:
        for p, q in (((0, 0, 0), d), (d, (0, 0, 0))):
            carried, stays = _masks(np.subtract(q, p))
            if (ent[around[q]][_bits(carried)][:, None] == ent[around[p]][~_bits(stays)][None, :]).any():
                return True
    return False


def _path_cells(lay, lvl, rng):
    """The scripted cell sequence around a cell A: A, A + d, A for every neighbour move d (each move followed by its
    reverse), oscillation A B A B (B a face and an edge neighbour), +2 on x and -2 on y, and A + x, A + 2x, A (a jump
    back to an earlier cell).  On hashed levels A is drawn until one of its moves carries a corner onto the entry of a
    leaving one."""
    res = lay.resolutions[lvl]
    A = rng.integers(2, res - 2, 3) if res > 4 else np.array([res // 2 - 1, res // 2, res // 2])
    while lvl >= lay.begin_fast_hash_level and not _carry_collides(lay, lvl, A):
        A = rng.integers(2, res - 2, 3)
    ex, ey = np.array([1, 0, 0]), np.array([0, 1, 0])
    seq = []
    for d in rng.permutation(sorted(MOVES)):
        seq += [A, A + d]
    seq.append(A)
    B, D = A + ex, A + np.array([1, -1, 0])
    seq += [B, A, B, D, A, D, A + 2 * ex, A, A - 2 * ey, A, A + ex, A + 2 * ex, A]
    return seq


def _scripted_path(lay, lvl, rng, nonneg):
    """The rows of one scripted path at level lvl: runs of 1 to 5 rows per visited cell, the first row of every third
    run on a face, and skipped rows (dy zero at lvl) inside runs and between runs.  The last row is a run's."""
    L = lay.levels
    rows = _Rows(L)
    for v, cell in enumerate(_path_cells(lay, lvl, rng)):
        if v and rng.random() < 0.25:                                                # between two runs
            _skip_row(rows, rng, L, lvl, v)
        k = int(rng.integers(1, 6))
        faces = np.zeros(k, bool)
        faces[0] = v % 3 == 0
        x = _cell_points(lay, lvl, np.tile(cell, (k, 1)), rng, faces, nonneg)
        skip_at = int(rng.integers(1, k)) if k > 1 and rng.random() < 0.3 else -1     # inside the run
        for j in range(k):
            if j == skip_at:
                _skip_row(rows, rng, L, lvl, v)
            rows.add(x[j], _other_zero(rng, L, lvl), v)
    return rows


def _skip_row(rows, rng, L, lvl, v):
    """One row that the walk at lvl must skip: zero at every level at a NaN position, or zero at lvl only at a random
    point of the box (another cell)."""
    if v % 2:
        rows.add(np.full(3, np.nan), np.ones(L, bool), -1)
    else:
        z = _other_zero(rng, L, lvl)
        z[:, lvl] = True
        rows.add(rng.random(3), z, -1)


def _edge_path(lay, lvl, rng, negative):
    """The box's corners at level lvl: x = 1 exactly (on dense levels a corner index past the level's size), the cells
    beyond it (grid coordinate up to res), mixed exact coordinates, x = 0 exactly and, when `negative`, cells at grid
    coordinate -1."""
    L = lay.levels
    s = lay.scales[lvl]
    g1 = int(np.floor(_f32_pos(1.0, s)))
    rows = _Rows(L)
    one, zero = np.ones(3, np.float32), np.zeros(3, np.float32)

    def cell(c, k, v):
        rows.add(_cell_points(lay, lvl, np.tile(c, (k, 1)), rng, np.zeros(k, bool), not negative),
                 _other_zero(rng, L, lvl, k), v)

    def exact(x, k, v):
        rows.add(np.tile(np.asarray(x, np.float32), (k, 1)), _other_zero(rng, L, lvl, k), v)

    G1 = np.full(3, g1)
    exact(one, 2, 0)
    cell(G1 + 1, 2, 1)
    exact(one, 1, 2)
    cell(G1 + np.array([1, 0, 0]), 1, 3)
    exact(one, 2, 4)
    cell(G1 + np.array([0, -1, 1]), 2, 5)
    exact([1, 0, 1], 1, 6)
    exact([0, 1, 0], 1, 7)
    exact([1, 1, 0], 1, 8)
    exact(zero, 2, 9)
    cell(np.array([1, 0, 0]), 2, 10)
    exact(zero, 1, 11)
    if negative:
        cell(np.array([-1, -1, -1]), 2, 12)
        exact(zero, 1, 13)
        cell(np.array([-1, 0, 0]), 1, 14)
        cell(np.array([0, -1, 0]), 2, 15)
        exact(zero, 1, 16)
    return rows


class Stream(NamedTuple):
    lay: object
    x: np.ndarray          # fp32 [n, 3]; NaN on rows whose dy is zero at every level
    dout: np.ndarray       # [n, L * 2], fp32 or fp16
    copies: list           # (scripted level, first row, end row) of every scripted path


@functools.lru_cache(maxsize=None)
def _stream(L, half):
    """For each scripted level: 16 scripted paths, the k-th starting at offset k of a lane's chunk, then one edge path.
    The rows between two paths repeat the last row of the first, so they extend its last run; a path is moved by whole
    chunks until every CTA boundary in it or before it falls inside a run."""
    lay = _layout(L)
    rng = np.random.default_rng(500 + L)
    out, copies, cur = _Rows(L), [], 0
    for lvl in _scripted_levels(lay):
        paths = [_scripted_path(lay, lvl, rng, nonneg=True) for _ in range(CHUNK)]
        paths.append(_edge_path(lay, lvl, rng, negative=not half))
        for k, path in enumerate(paths):
            px, pz, prun = path.arrays()
            prun = np.where(prun >= 0, prun + 1000 * len(copies), -1)     # run ids unique over the stream
            last = (out.x[-1][-1], out.zero[-1][-1], out.run[-1][-1]) if out.x else None
            start = -(-cur // CHUNK) * CHUNK + k
            while True:
                run = np.concatenate([[last[2] if last else -1], np.full(start - cur, last[2] if last else -1), prun])
                if all(run[b - cur] == run[b - cur + 1] >= 0                 # run[i] is row cur - 1 + i
                       for b in range(max(CTA, -(-cur // CTA) * CTA), start + len(px), CTA)):
                    break
                start += CHUNK
            if start > cur:
                out.add(np.tile(last[0], (start - cur, 1)), last[1], last[2])
            out.add(px, pz, prun)
            copies.append((lvl, start, start + len(px)))
            cur = start + len(px)
    x, zero, _ = out.arrays()
    n = len(x)
    d = rng.standard_normal((n, L, 2)).astype(np.float32)
    d[zero] = 0.0
    part = (rng.random((n, L)) < 0.05) & ~zero                    # dy = (a, 0) or (0, a) still contributes
    d[part, rng.integers(0, 2, int(part.sum()))] = 0.0
    d = d.reshape(n, L * 2)
    return Stream(lay, x, d.astype(np.float16) if half else d, copies)


@functools.lru_cache(maxsize=4)
def _table(L, half):
    t = np.random.default_rng(600 + L).standard_normal(_layout(L).total_param_size).astype(np.float32) * 0.1
    return t.astype(np.float16) if half else t


def _x_fwd(s):
    """The forward computes every row (it has no skip): the NaN rows of the stream are moved into the box."""
    return np.where(np.isfinite(s.x), s.x, np.float32(0.5))


# ---- what the streams contain (CPU) -------------------------------------------------------------------------------------
def _masks(d):
    """cell_step of hash.cu for one move d: (carried corners of the new cell, corners of the old cell that stay)."""
    low = (0x55, 0x33, 0x0F)
    carried = stays = 0xFF
    for k in range(3):
        lo, hi = low[k], ~low[k] & 0xFF
        carried &= {0: 0xFF, 1: lo, -1: hi}.get(int(d[k]), 0)
        stays &= {0: 0xFF, 1: hi, -1: lo}.get(int(d[k]), 0)
    return carried, stays


@functools.lru_cache(maxsize=256)
def _bits(m):
    return np.array([(m >> c) & 1 for c in range(8)], bool)


def _level_rows(s, lvl, half):
    """Per row at lvl: live (dy != 0), signed grid coordinate, fraction and the 8 corner entries."""
    lay = s.lay
    n = len(s.x)
    live = (np.asarray(s.dout).reshape(n, lay.levels, 2)[:, lvl] != 0).any(1)
    xf = np.where(np.isfinite(s.x), s.x, np.float32(0.5))
    g, frac = grid_cell(xf, lay, lvl, half)
    ent = np.stack([corner_entries(lay, lvl, g, c) for c in range(8)], 1)
    return live, g, g.view(np.int32).astype(np.int64), frac, ent


def _census(s, lvl, half):
    """What the backward's walk at lvl meets in the stream, counted from the positions and dL/dout alone."""
    lay = s.lay
    n = len(s.x)
    live, g, gs, frac, ent = _level_rows(s, lvl, half)
    c = {}
    rows = np.flatnonzero(live)
    a, b = rows[:-1], rows[1:]
    # consecutive live rows of one lane: moves, and the move sequence of each lane
    lane = a // CHUNK == b // CHUNK
    d = (g[b] - g[a]).view(np.int32).astype(np.int64)
    mv = np.flatnonzero(lane & (d != 0).any(1))
    dm, ch = d[mv], a[mv] // CHUNK
    nb = np.abs(dm).max(1) == 1
    c["moves"] = {tuple(v) for v in dm[nb]}
    same2 = ch[1:] == ch[:-1]
    rev = same2 & nb[:-1] & (dm[1:] == -dm[:-1]).all(1)
    c["reversed"] = {tuple(v) for v in dm[:-1][rev]}
    same3 = same2[1:] & same2[:-1]
    c["oscillation"] = int((same3 & rev[:-1] & rev[1:]).sum())
    c["two_on_one_axis"] = int((np.sort(np.abs(dm), 1) == [0, 0, 2]).all(1).sum())
    c["jump_back"] = int((same3 & (dm[:-2] + dm[1:-1] + dm[2:] == 0).all(1) & ~nb[2:]).sum())
    # skipped rows between two live rows of one lane: inside a run (same cell on both sides) or between runs
    idx = np.arange(n)
    prev = np.maximum.accumulate(np.where(live, idx, -1))
    nxt = np.minimum.accumulate(np.where(live, idx, n)[::-1])[::-1]
    sk = np.flatnonzero(~live)
    sk = sk[(prev[sk] >= 0) & (nxt[sk] < n)]
    sk = sk[(prev[sk] // CHUNK == sk // CHUNK) & (nxt[sk] // CHUNK == sk // CHUNK)]
    inside = (g[prev[sk]] == g[nxt[sk]]).all(1)
    c["skip_in_run"], c["skip_between_runs"] = int(inside.sum()), int((~inside).sum())
    c["skip_nan"] = int((~np.isfinite(s.x[sk]).all(1)).sum())
    dy = np.asarray(s.dout).reshape(n, lay.levels, 2)
    c["zero_elsewhere_only"] = int((live & ~(dy != 0).any(2).all(1)).sum())
    # runs across a lane's chunk boundary and across a CTA boundary
    r = np.arange(CHUNK, n, CHUNK)
    run_cross = r[live[r - 1] & live[r] & (g[r - 1] == g[r]).all(1)]
    c["run_across_chunk"] = int((run_cross % CTA != 0).sum())
    c["run_across_cta"] = run_cross[run_cross % CTA == 0].tolist()
    # faces and the box edge, on the rows the walk scatters
    L_ = live & np.isfinite(s.x).all(1)
    c["face"] = int((L_[:, None] & (frac == 0)).any(1).sum())
    c["x0"] = int((L_[:, None] & (s.x == 0)).any(1).sum())
    c["x1"] = int((L_[:, None] & (s.x == 1)).any(1).sum())
    c["g_negative"] = int((L_[:, None] & (gs < 0)).any(1).sum())
    c["g_past_res"] = int((L_[:, None] & (gs >= lay.resolutions[lvl])).any(1).sum())
    # neighbour moves: carried / leaving corners, leaving x-pairs merged into one reduction, and entry collisions
    nbm = mv[nb]
    old, new = ent[a[nbm]], ent[b[nbm]]
    masks = [_masks(v) for v in d[nbm]]
    carried = np.array([_bits(m[0]) for m in masks]).reshape(-1, 8)
    leaving = ~np.array([_bits(m[1]) for m in masks]).reshape(-1, 8)
    pair = leaving[:, 0::2] & leaving[:, 1::2] & ((old[:, 0::2] ^ old[:, 1::2]) == 1)
    c["merged_pairs"] = int(pair.sum())
    c["carried_corners"] = int(carried.sum())
    if lvl >= lay.begin_fast_hash_level:
        e = np.sort(ent[live], 1)
        c["cell_collision"] = int((e[:, 1:] == e[:, :-1]).any(1).sum())
        eq = (new[:, :, None] == old[:, None, :]) & carried[:, :, None] & leaving[:, None, :]
        c["carried_leaving_collision"] = int(eq.any((1, 2)).sum())
    else:
        res = np.uint32(lay.resolutions[lvl])
        wrap = np.zeros(n, bool)
        for k in range(8):
            p = [g[:, dd] + np.uint32((k >> dd) & 1) for dd in range(3)]
            wrap |= (p[0] + p[1] * res + p[2] * (res * res)) >= np.uint32(lay.map_sizes[lvl])
        c["dense_wrap"] = int((wrap & L_).sum())
    return c


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("L", LEVEL_COUNTS)
def test_walk_streams_exercise_every_path(L, half):
    """Every category the file's docstring lists occurs at every scripted level, inside one lane's walk where it is a
    walk property; CTA boundaries 512 and 1024 fall inside runs (the n = 513 and 1025 prefixes cut there)."""
    s = _stream(L, half)
    lay = s.lay
    assert len(s.x) > 2 * CTA + 1
    across = set()
    for lvl in _scripted_levels(lay):
        c = _census(s, lvl, half)
        what = f"L={L} level {lvl}"
        assert c["moves"] == MOVES, f"{what}: moves never seen {MOVES - c['moves']}"
        assert c["reversed"] == MOVES, f"{what}: moves never reversed {MOVES - c['reversed']}"
        for k in ("oscillation", "two_on_one_axis", "jump_back", "skip_in_run", "skip_between_runs", "skip_nan",
                  "run_across_chunk", "face", "x0", "x1", "g_past_res", "merged_pairs", "carried_corners"):
            assert c[k] > 0, f"{what}: no {k}"
        assert c["zero_elsewhere_only"] > 0 or L == 1, f"{what}: no row zero at other levels only"
        assert c["run_across_cta"], f"{what}: no run across a CTA boundary"
        across.update(c["run_across_cta"])
        assert (c["g_negative"] > 0) == (not half), f"{what}: g_negative {c['g_negative']}"
        if lvl >= lay.begin_fast_hash_level:
            assert c["cell_collision"] > 0 and c["carried_leaving_collision"] > 0, f"{what}: {c}"
        else:
            assert c["dense_wrap"] > 0, f"{what}: no corner index past the dense level's size"
    assert {CTA, 2 * CTA} <= across
    starts = {(lvl, a % CHUNK) for lvl, a, _ in s.copies}
    assert starts == {(lvl, o) for lvl in _scripted_levels(lay) for o in range(CHUNK)}


# ---- the check has teeth (CPU) ------------------------------------------------------------------------------------------
def _walk_flushes(x, dout, lay, lvl, half):
    """hash_bwd_kernel's walk at lvl restated in Python with fp64 sums: per 16-row chunk, over the rows whose dy is not
    zero at lvl, a cell change flushes the old cell's corners that the new cell does not share and carries the others;
    the chunk's end flushes all 8.  Returns one record per flushed corner: (entry, value [2], carried: the value holds
    rows of an earlier cell, at_move: flushed at a cell change, partner: index of the other record of a merged x-pair
    reduction or -1)."""
    n = len(x)
    dy = np.asarray(dout).reshape(n, lay.levels, 2)[:, lvl].astype(np.float64)
    live = (dy != 0).any(1)
    g, frac = grid_cell(np.where(live[:, None], x, np.float32(0.5)), lay, lvl, half)
    ent = np.stack([corner_entries(lay, lvl, g, c) for c in range(8)], 1)
    w = np.ones((n, 8), np.float32)
    for c in range(8):
        for d in range(3):
            w[:, c] = w[:, c] * (frac[:, d] if c & (1 << d) else np.float32(1) - frac[:, d])
    rec = []

    def flush(e, acc, was, leaving, at_move):
        for c in range(0, 8, 2):
            out0, out1 = (leaving >> c) & 1, (leaving >> (c + 1)) & 1
            merged = out0 and out1 and (e[c] ^ e[c + 1]) == 1
            for k, out in ((c, out0), (c + 1, out1)):
                if out:
                    rec.append([int(e[k]), acc[k].copy(), bool(was[k]), at_move, -1])
            if merged:
                rec[-1][4], rec[-2][4] = len(rec) - 2, len(rec) - 1

    for c0 in range(0, n, CHUNK):
        pg, acc, was = None, np.zeros((8, 2)), np.zeros(8, bool)
        for r in range(c0, min(c0 + CHUNK, n)):
            if not live[r]:
                continue
            if pg is None or (g[r] != g[pg]).any():
                nacc, nwas = np.zeros((8, 2)), np.zeros(8, bool)
                if pg is not None:
                    d = (g[r] - g[pg]).view(np.int32)
                    carried, stays = _masks(d)
                    flush(ent[pg], acc, was, ~stays & 0xFF, True)
                    for c in range(8):
                        if (carried >> c) & 1:      # corner c of the new cell is corner c + d of the old one
                            o = sum((((c >> k) & 1) + int(d[k])) << k for k in range(3))
                            nacc[c], nwas[c] = acc[o], True
                pg, acc, was = r, nacc, nwas
            acc += w[r].astype(np.float64)[:, None] * dy[r]
        if pg is not None:
            flush(ent[pg], acc, was, 0xFF, False)
    return rec


def test_check_scatter_rejects_seeded_walk_faults():
    """The fp64 scatter rounded to fp32 passes _check_scatter; with one carried corner's run moved to the neighbouring
    entry, one leaving corner dropped, or a merged x-pair's two values swapped, it is rejected.  The walk restated
    here is first shown to partition the fp64 scatter exactly."""
    s = _stream(16, False)
    lay = s.lay
    lvl = lay.begin_fast_hash_level
    _, a, b = next(c for c in s.copies if c[0] == lvl)
    a -= a % CHUNK
    x, dout = s.x[a:b], s.dout[a:b]
    ref, mag, cnt = np_hash_bwd_f64(x, dout, lay, False, [lvl])
    lo, hi = _level_slice(lay, lvl, lvl + 1)
    rec = _walk_flushes(x, dout, lay, lvl, False)
    total = np.zeros_like(ref).reshape(-1, 2)
    for e, v, *_ in rec:
        total[e] += v
    np.testing.assert_allclose(total.reshape(-1), ref, rtol=1e-12, atol=1e-12)
    prefill = (np.random.default_rng(7).standard_normal(ref.size) * 1e-2).astype(np.float32)

    def scattered(delta):
        return (prefill.astype(np.float64) + ref + delta).astype(np.float32)

    _check_scatter(scattered(0.0), prefill, ref, mag, cnt, lo, hi, "fp64 scatter")
    faults = {}
    i = max((i for i, r in enumerate(rec) if r[2]), key=lambda i: np.abs(rec[i][1]).max())
    e, v = rec[i][0], rec[i][1]
    delta = np.zeros((ref.size // 2, 2))
    delta[e] -= v
    delta[e ^ 1] += v
    faults["carried corner moved to the neighbouring entry"] = delta
    i = max((i for i, r in enumerate(rec) if r[3]), key=lambda i: np.abs(rec[i][1]).max())
    delta = np.zeros((ref.size // 2, 2))
    delta[rec[i][0]] -= rec[i][1]
    faults["leaving corner dropped"] = delta
    i = max((i for i, r in enumerate(rec) if r[4] >= 0), key=lambda i: np.abs(rec[i][1] - rec[rec[i][4]][1]).max())
    j = rec[i][4]
    delta = np.zeros((ref.size // 2, 2))
    delta[rec[i][0]] += rec[j][1] - rec[i][1]
    delta[rec[j][0]] += rec[i][1] - rec[j][1]
    faults["merged x-pair swapped"] = delta
    for what, delta in faults.items():
        assert np.abs(delta).max() > 1e-2, what
        with pytest.raises(AssertionError):
            _check_scatter(scattered(delta.reshape(-1)), prefill, ref, mag, cnt, lo, hi, what)


# ---- forward and backward on the GPU --------------------------------------------------------------------------------------
def _buffer(rows, cols, dtype, fill, view):
    """(allocation, [rows, cols] matrix in it): at element 0, or with `view` one entry (2 elements) past the 16-byte
    aligned start, which keeps entry alignment and makes the kernels take their scalar branches."""
    flat = torch.full((rows * cols + 2,), fill, device=DEV, dtype=dtype)
    m = (flat[2:] if view else flat[:-2]).view(rows, cols)
    assert flat.data_ptr() % 16 == 0 and (m.data_ptr() % 16 != 0) == view
    return flat, m


def _cases():
    return [pytest.param(L, False, id=f"L{L}") for L in LEVEL_COUNTS] + [pytest.param(16, True, id="L16-view")]


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("L,view", _cases())
def test_walk_fwd_bit_exact(lib, oracle, L, view, half):
    """Every prefix n of the stream, bit for bit against the oracle; rows at or past n and the element before an
    offset view keep the sentinel."""
    s = _stream(L, half)
    lay, cl = s.lay, s.lay.as_ctypes()
    x = _x_fwd(s)
    table = _table(L, half)
    ref = oracle.hash_encode_fwd(x, table, lay)
    dt, vt = (torch.float16, np.uint16) if half else (torch.float32, np.uint32)
    t_x, t_tab = T(x), T(table)
    for n in N_ROWS + (len(x),):
        flat, out = _buffer(n + 64, lay.out_dim, dt, SENTINEL, view)
        chk(lib.ngp_hash_encode_fwd(P(t_x), P(t_tab), C.byref(cl), P(out), F16 if half else F32, n, ST()))
        got = N(out)
        assert np.array_equal(got[:n].view(vt), ref[:n].view(vt)), f"n={n}: rows differ from the oracle"
        written = np.flatnonzero((got[n:] != SENTINEL).any(1))
        assert written.size == 0, f"n={n}: row {n + written[0]} at or past n was written"
        guard = N(flat)[:2] if view else N(flat)[-2:]
        assert (guard == SENTINEL).all(), f"n={n}: an element outside out was written"


def _dout_buffer(dout, view):
    flat, m = _buffer(dout.shape[0], dout.shape[1], torch.float16 if dout.dtype == np.float16 else torch.float32,
                      0.0, view)
    m.copy_(T(dout))
    return flat, m


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("L,view", _cases())
def test_walk_bwd_fp64_bound(lib, L, view, half):
    """Every prefix n of the stream against the fp64 scatter: every entry within the any-order bound, entries no row
    reaches bit-unchanged."""
    s = _stream(L, half)
    lay, cl = s.lay, s.lay.as_ctypes()
    t_x = T(s.x)
    _, t_d = _dout_buffer(s.dout, view)
    prefill = (np.random.default_rng(700 + L).standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    for n in N_ROWS + (len(s.x),):
        g = T(prefill)
        chk(lib.ngp_hash_encode_bwd(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n, ST()))
        ref, mag, cnt = np_hash_bwd_f64(s.x[:n], s.dout[:n], lay, half, range(lay.levels))
        if n == len(s.x):
            assert cnt.max() > 8
        _check_scatter(N(g), prefill, ref, mag, cnt, 0, lay.total_param_size, f"n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("L", [5, 16])
def test_walk_dyn_row_count(lib, oracle, L, half):
    """ngp_hash_encode_fwd_dyn and _bwd_dyn with the row count on the device: rows [0, min(n_max, max(n_dev, 0)))
    as the plain entries compute them, rows at or past the count untouched (forward: the sentinel; backward: no
    contribution)."""
    s = _stream(L, half)
    lay, cl = s.lay, s.lay.as_ctypes()
    n_max = 1025
    assert len(s.x) >= n_max + PAD
    x = _x_fwd(s)
    ref = oracle.hash_encode_fwd(x[:n_max], _table(L, half), lay)
    dt, vt = (torch.float16, np.uint16) if half else (torch.float32, np.uint32)
    tag = F16 if half else F32
    t_xf, t_tab, t_x, t_d = T(x), T(_table(L, half)), T(s.x), T(s.dout)
    prefill = (np.random.default_rng(800 + L).standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    for nd in n_dev_cases(n_max):
        m, t_nd = rows_of(nd, n_max), i32(nd)     # (named: a temporary's memory could be reused before the launch)
        out = torch.full((n_max + PAD, lay.out_dim), SENTINEL, device=DEV, dtype=dt)
        chk(lib.ngp_hash_encode_fwd_dyn(P(t_xf), P(t_tab), C.byref(cl), P(out), tag, n_max, P(t_nd), None, ST()))
        got = N(out)
        assert np.array_equal(got[:m].view(vt), ref[:m].view(vt)), f"n_dev={nd}: rows differ from the oracle"
        assert (got[m:] == SENTINEL).all(), f"n_dev={nd}: a row at or past the count was written"
        g = T(prefill)
        chk(lib.ngp_hash_encode_bwd_dyn(P(t_x), P(t_d), tag, C.byref(cl), P(g), n_max, P(t_nd), None, ST()))
        ref_b = np_hash_bwd_f64(s.x[:m], s.dout[:m], lay, half, range(lay.levels))
        _check_scatter(N(g), prefill, *ref_b, 0, lay.total_param_size, f"n_dev={nd}")


def _walk_ranges(L, half):
    """Every [a, b) at L = 5; at L = 16 the ranges whose ends are not both multiples of kVec (2 fp32, 4 fp16), where
    the vector staging of dL/dout keeps only the columns inside the range."""
    if L == 5:
        return [(a, b) for a in range(5) for b in range(a + 1, 6)]
    kvec = 4 if half else 2
    cand = sorted(set(_level_ranges(_layout(L)).values()) | {(2, 7), (6, 10)})
    return [(a, b) for a, b in cand if a % kvec or b % kvec]


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("L", [5, 16])
def test_walk_bwd_levels_fp64_bound(lib, L, half):
    """ngp_hash_encode_bwd_levels on the whole stream: the range's levels within the bound, every other level's slice
    bit-unchanged."""
    s = _stream(L, half)
    lay, cl = s.lay, s.lay.as_ctypes()
    t_x, t_d = T(s.x), T(s.dout)
    n = len(s.x)
    ref, mag, cnt = np_hash_bwd_f64(s.x, s.dout, lay, half, range(lay.levels))
    prefill = (np.random.default_rng(900 + L).standard_normal(lay.total_param_size) * 1e-2).astype(np.float32)
    ranges = _walk_ranges(L, half)
    assert len(ranges) >= (15 if L == 5 else 4)
    for a, b in ranges:
        g = T(prefill)
        chk(lib.ngp_hash_encode_bwd_levels(P(t_x), P(t_d), F16 if half else F32, C.byref(cl), P(g), n, None, None,
                                           a, b, None, ST()))
        lo, hi = _level_slice(lay, a, b)
        _check_scatter(N(g), prefill, ref, mag, cnt, lo, hi, f"levels [{a},{b})")
