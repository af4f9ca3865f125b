"""Numpy restatement of the marching-cubes contract (DESIGN.md §6g), vectorised, in fp32 with every operation rounded
on its own (numpy never fuses a multiply and an add), so the sm_90a kernels can be compared with it exactly.

The case table comes from scripts/gen_mc_table.py, the generator of the committed header; everything else (lattice
coordinates, interpolation, normals, vertex and face order) is written here from the contract, not from the kernels.
Also holds the mesh checks the tests use: edge incidence, Euler characteristic, signed volume, components.
"""
from __future__ import annotations

import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def load_generator():
    spec = importlib.util.spec_from_file_location("gen_mc_table", os.path.join(ROOT, "scripts", "gen_mc_table.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_GEN = load_generator()
TABLE = _GEN.build_table()
EDGES = _GEN.EDGES                  # [(corner_a, corner_b, axis)] * 12
MAX_TRIS = max(len(t) for t in TABLE)
TRI_EDGES = np.full((256, 3 * MAX_TRIS), -1, np.int64)
for _c, _tris in enumerate(TABLE):
    _flat = [e for t in _tris for e in t]
    TRI_EDGES[_c, :len(_flat)] = _flat
TRI_COUNT = np.array([len(t) for t in TABLE], np.int64)


def spacing(n, bound):
    """s = f_div(2b, N - 1)."""
    return f32(f32(2.0) * f32(bound)) / f32(n - 1)


def node_coords(n, bound):
    """fp32 [n]: f_add(-b, f_mul((float)i, s))."""
    s = spacing(n, bound)
    return f32(-f32(bound)) + np.arange(n, dtype=f32) * s


def gradient(lat):
    """fp32 [N, N, N, 3] in units of 1/spacing: (v[i+1] - v[i-1]) * 0.5 inside, one-sided differences on the
    border (the spacing is the same on every axis and the normal is normalised, so it is left out)."""
    n = lat.shape[0]
    g = np.empty(lat.shape + (3,), f32)
    for axis in range(3):
        v = np.moveaxis(lat, axis, 0)
        d = np.empty_like(v)
        if n > 2:
            d[1:-1] = (v[2:] - v[:-2]) * f32(0.5)
        d[0] = v[1] - v[0]
        d[-1] = v[-1] - v[-2]
        g[..., axis] = np.moveaxis(d, 0, axis)
    return g


def marching_cubes(lat, threshold, bound):
    """(vertices fp32 [V, 3], normals fp32 [V, 3], faces int32 [F, 3]) of the fp32 lattice [N, N, N] (indexed
    [ix, iy, iz], z fastest) over [-bound, bound]^3 at `threshold`."""
    lat = np.ascontiguousarray(lat, dtype=f32)
    n = lat.shape[0]
    assert lat.shape == (n, n, n) and n >= 2
    tau = f32(threshold)
    s = spacing(n, bound)
    xs = node_coords(n, bound)
    inside = lat > tau

    # crossing edges, ordered by edge id = node_linear * 3 + axis
    ids, va, vb, nodes, axes = [], [], [], [], []
    for axis in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[axis] = slice(0, n - 1)
        hi[axis] = slice(1, n)
        cross = inside[tuple(lo)] != inside[tuple(hi)]
        idx = np.argwhere(cross)                       # node a of each crossing edge
        lin = (idx[:, 0] * n + idx[:, 1]) * n + idx[:, 2]
        ids.append(lin * 3 + axis)
        nodes.append(idx)
        axes.append(np.full(len(idx), axis, np.int64))
        b = idx.copy()
        b[:, axis] += 1
        va.append(lat[idx[:, 0], idx[:, 1], idx[:, 2]])
        vb.append(lat[b[:, 0], b[:, 1], b[:, 2]])
    ids = np.concatenate(ids)
    order = np.argsort(ids, kind="stable")
    ids = ids[order]
    va = np.concatenate(va)[order]
    vb = np.concatenate(vb)[order]
    nodes = np.concatenate(nodes)[order]
    axes = np.concatenate(axes)[order]
    nv = len(ids)

    t = (tau - va) / (vb - va)
    verts = np.stack([xs[nodes[:, 0]], xs[nodes[:, 1]], xs[nodes[:, 2]]], axis=1).astype(f32)
    rows = np.arange(nv)
    verts[rows, axes] = verts[rows, axes] + t * s

    if nv:
        g = gradient(lat)
        nb = nodes.copy()
        nb[rows, axes] += 1
        ga = g[nodes[:, 0], nodes[:, 1], nodes[:, 2]]
        gb = g[nb[:, 0], nb[:, 1], nb[:, 2]]
        m = ga + t[:, None] * (gb - ga)
        length = np.sqrt((m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1]) + m[:, 2] * m[:, 2])
        zero = length == 0
        with np.errstate(divide="ignore", invalid="ignore"):
            normals = -(m / np.where(zero, f32(1), length)[:, None])
        normals[zero] = (0, 0, 1)
        normals = normals.astype(f32)
    else:
        normals = np.zeros((0, 3), f32)

    # faces: cells in linear order, then the table's order within the cell
    c = n - 1
    case = np.zeros((c, c, c), np.int64)
    for k in range(8):
        dx, dy, dz = k & 1, k >> 1 & 1, k >> 2 & 1
        case |= inside[dx:dx + c, dy:dy + c, dz:dz + c].astype(np.int64) << k
    cells = np.argwhere(TRI_COUNT[case] > 0)          # lexicographic = cell linear order
    if len(cells) == 0:
        return verts, normals, np.zeros((0, 3), np.int32)
    cc = case[cells[:, 0], cells[:, 1], cells[:, 2]]
    te = TRI_EDGES[cc]                                 # [M, 3 * MAX_TRIS]
    valid = te >= 0
    cell_of = np.broadcast_to(np.arange(len(cells))[:, None], te.shape)[valid]
    e = te[valid]
    corner = np.array([a for a, _, _ in EDGES])[e]
    axis = np.array([ax for _, _, ax in EDGES])[e]
    node = cells[cell_of] + np.stack([corner & 1, corner >> 1 & 1, corner >> 2 & 1], axis=1)
    eid = ((node[:, 0] * n + node[:, 1]) * n + node[:, 2]) * 3 + axis
    vid = np.searchsorted(ids, eid)
    assert np.all(ids[vid] == eid)
    faces = vid.reshape(-1, 3).astype(np.int32)
    return verts, normals, faces


# ---- mesh checks -------------------------------------------------------------------------------------------------
def edge_incidence(faces):
    """(face count of each undirected edge, face count of each directed edge), over the edges the faces use."""
    f = faces.astype(np.int64)
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    m = int(f.max()) + 1 if len(f) else 1
    _, dcount = np.unique(a * m + b, return_counts=True)
    _, ucount = np.unique(np.minimum(a, b) * m + np.maximum(a, b), return_counts=True)
    return ucount, dcount


def is_closed_oriented(faces):
    ucount, dcount = edge_incidence(faces)
    return bool(np.all(ucount == 2) and np.all(dcount == 1))


def euler_characteristic(n_vertices, faces):
    ucount, _ = edge_incidence(faces)
    return int(n_vertices) - len(ucount) + len(faces)


def signed_volume(verts, faces):
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def components(n_vertices, faces):
    """Number of connected components of the vertices the faces use."""
    parent = np.arange(n_vertices)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for a, b, c in faces:
        ra, rb, rc = find(a), find(b), find(c)
        parent[rb] = ra
        parent[find(rc)] = ra
    used = np.unique(faces)
    return len({find(v) for v in used})


# ---- analytic fields ---------------------------------------------------------------------------------------------
def grid_points(n, bound):
    x = node_coords(n, bound).astype(np.float64)
    return np.meshgrid(x, x, x, indexing="ij")


def sphere_field(n, bound, radius, center=(0.0, 0.0, 0.0)):
    """fp32 lattice radius - |x - center|: inside (> 0) within the sphere."""
    x, y, z = grid_points(n, bound)
    r = np.sqrt((x - center[0]) ** 2 + (y - center[1]) ** 2 + (z - center[2]) ** 2)
    return (radius - r).astype(f32)


def torus_field(n, bound, major, minor):
    x, y, z = grid_points(n, bound)
    q = np.sqrt(x ** 2 + y ** 2) - major
    return (minor - np.sqrt(q ** 2 + z ** 2)).astype(f32)


def random_field(n, seed, threshold=0.0, block=1):
    """Seeded lattice with an outside border: values in {threshold - 1, threshold, threshold + 1} and uniform noise,
    so exact-threshold nodes (outside: v > tau fails) are common.  block > 1 repeats each value over block^3 nodes
    (fewer crossings at large n)."""
    rng = np.random.default_rng(seed)
    m = -(-n // block)
    lat = rng.uniform(-1, 1, (m, m, m)).astype(f32) + f32(threshold)
    pick = rng.random((m, m, m))
    lat[pick < 0.2] = f32(threshold)
    lat[(pick >= 0.2) & (pick < 0.3)] = f32(threshold + 1)
    if block > 1:
        lat = np.ascontiguousarray(lat.repeat(block, 0).repeat(block, 1).repeat(block, 2)[:n, :n, :n])
    lat[0, :, :] = lat[-1, :, :] = lat[:, 0, :] = lat[:, -1, :] = lat[:, :, 0] = lat[:, :, -1] = f32(threshold - 1)
    return lat


def read_ply(path):
    """(vertices fp32 [V, 3], normals fp32 [V, 3], colours uint8 [V, 3], faces int64 [F, 3]) of a binary
    little-endian PLY with write_ply's layout; raises on anything else."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").splitlines()
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0", lines[:2]
    nv = nf = None
    props = []
    for ln in lines[2:]:
        w = ln.split()
        if w[:2] == ["element", "vertex"]:
            nv = int(w[2])
        elif w[:2] == ["element", "face"]:
            nf = int(w[2])
        elif w[0] == "property":
            props.append(" ".join(w[1:]))
    assert props == ["float x", "float y", "float z", "float nx", "float ny", "float nz", "uchar red", "uchar green",
                     "uchar blue", "list uchar uint32 vertex_indices"], props
    vt = np.dtype([("p", "<f4", (3,)), ("n", "<f4", (3,)), ("c", "u1", (3,))])
    ft = np.dtype([("k", "u1"), ("i", "<u4", (3,))])
    verts = np.frombuffer(data, vt, nv, end)
    faces = np.frombuffer(data, ft, nf, end + nv * vt.itemsize)
    assert end + nv * vt.itemsize + nf * ft.itemsize == len(data), "trailing bytes"
    assert np.all(faces["k"] == 3)
    return verts["p"].copy(), verts["n"].copy(), verts["c"].copy(), faces["i"].astype(np.int64)
