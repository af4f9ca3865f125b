"""CPU checks of the mesh export (DESIGN.md §6g): the generated case table, the numpy restatement of the contract on
analytic fields, the PLY writer, the --mesh_* flags and the C-ABI argument checks."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import mc_ref as M
from conftest import ROOT

GEN = M.load_generator()


# ---- the case table ----------------------------------------------------------------------------------------------
def test_generator_reproduces_committed_header():
    with open(os.path.join(ROOT, "taichi_nerfs_b200", "csrc", "mc_table.cuh")) as f:
        assert f.read() == GEN.render_header()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_mc_table.py"), "--check"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_empty_cases():
    assert M.TABLE[0] == [] and M.TABLE[255] == []


def _crossing_edges(case):
    return {i for i, (a, b, _) in enumerate(GEN.EDGES) if (case >> a & 1) != (case >> b & 1)}


@pytest.mark.parametrize("case", range(256))
def test_case_uses_exactly_the_crossing_edges(case):
    used = {e for tri in M.TABLE[case] for e in tri}
    assert used == _crossing_edges(case)
    for tri in M.TABLE[case]:
        assert len(set(tri)) == 3


def _face_rule(case, ring):
    """Restated face rule: segments between crossing edges, an ambiguous face cutting off each inside corner."""
    inside = [bool(case >> c & 1) for c in ring]
    side = [GEN.edge_of(ring[i], ring[(i + 1) % 4]) for i in range(4)]
    cross = [i for i in range(4) if inside[i] != inside[(i + 1) % 4]]
    if len(cross) == 2:
        return {frozenset((side[cross[0]], side[cross[1]]))}
    if len(cross) == 4:
        return {frozenset((side[(i - 1) % 4], side[i])) for i in range(4) if inside[i]}
    return set()


@pytest.mark.parametrize("case", range(256))
def test_boundary_is_the_face_rule(case):
    """The edges that border one triangle of the case lie on cube faces and are the face rule's segments, face by
    face; every other edge borders two triangles of the case with opposite directions."""
    directed = {}
    for a, b, c in M.TABLE[case]:
        for p, q in ((a, b), (b, c), (c, a)):
            directed[(p, q)] = directed.get((p, q), 0) + 1
    assert all(v == 1 for v in directed.values())
    boundary = {frozenset(k) for k in directed if (k[1], k[0]) not in directed}
    want = set()
    for face in GEN.FACES:
        segs = _face_rule(case, face[2])
        on_face = {GEN.edge_of(face[2][i], face[2][(i + 1) % 4]) for i in range(4)}
        assert {s for s in boundary if s <= on_face} == segs, face
        want |= segs
    assert boundary == want


# ---- the restatement on analytic fields ----------------------------------------------------------------------------
def test_sphere():
    n, bound, r = 64, 1.0, 0.6
    v, nrm, f = M.marching_cubes(M.sphere_field(n, bound, r), 0.0, bound)
    ucount, dcount = M.edge_incidence(f)
    assert np.all(ucount == 2) and np.all(dcount == 1)
    assert M.euler_characteristic(len(v), f) == 2
    vol = 4 / 3 * np.pi * r ** 3
    assert abs(M.signed_volume(v, f) - vol) < 0.01 * vol
    dist = np.linalg.norm(v.astype(np.float64), axis=1)
    assert np.abs(dist - r).max() < M.spacing(n, bound)
    # normals are unit and point outward
    assert np.allclose(np.linalg.norm(nrm, axis=1), 1, atol=1e-6)
    assert np.all(np.einsum("ij,ij->i", nrm, v / dist[:, None]) > 0.99)


def test_torus():
    v, _, f = M.marching_cubes(M.torus_field(64, 1.0, 0.5, 0.2), 0.0, 1.0)
    assert M.is_closed_oriented(f)
    assert M.euler_characteristic(len(v), f) == 0
    assert M.signed_volume(v, f) > 0


def test_two_spheres():
    a = M.sphere_field(48, 1.0, 0.3, (-0.45, 0.0, 0.0))
    b = M.sphere_field(48, 1.0, 0.3, (0.45, 0.1, 0.0))
    v, _, f = M.marching_cubes(np.maximum(a, b), 0.0, 1.0)
    assert M.is_closed_oriented(f)
    assert M.components(len(v), f) == 2
    assert M.euler_characteristic(len(v), f) == 4


@pytest.mark.parametrize("seed", range(12))
def test_random_fields_closed_and_oriented(seed):
    lat = M.random_field(17, seed, threshold=0.25)
    assert np.sum(lat == np.float32(0.25)) > 0
    v, nrm, f = M.marching_cubes(lat, 0.25, 0.5)
    assert len(f) > 0
    assert M.is_closed_oriented(f)
    assert np.all(np.isfinite(v)) and np.all(np.isfinite(nrm))
    assert np.all(np.abs(v) <= 0.5)


def test_lattice_coordinates():
    x = M.node_coords(17, 0.5)
    assert x[0] == np.float32(-0.5) and x[8] == 0 and x[-1] == np.float32(0.5)


# ---- PLY ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_faces", [0, 5])
def test_write_ply_round_trip(tmp_path, n_faces):
    torch = pytest.importorskip("torch")
    from taichi_nerfs_b200.mesh import Mesh, write_ply
    rng = np.random.default_rng(n_faces)
    nv = 7
    v = rng.standard_normal((nv, 3)).astype(np.float32)
    nrm = rng.standard_normal((nv, 3)).astype(np.float32)
    col = rng.random((nv, 3)).astype(np.float32)
    col[0] = (0, 1, 0.5)
    f = rng.integers(0, nv, (n_faces, 3)).astype(np.int32)
    path = str(tmp_path / "m.ply")
    write_ply(path, Mesh(*(torch.from_numpy(a) for a in (v, nrm, col, f))))
    rv, rn, rc, rf = M.read_ply(path)
    assert np.array_equal(rv, v) and np.array_equal(rn, nrm) and np.array_equal(rf, f)
    assert np.array_equal(rc, np.rint(col * 255).astype(np.uint8))
    assert tuple(rc[0]) == (0, 255, 128)


def test_write_ply_empty(tmp_path):
    torch = pytest.importorskip("torch")
    from taichi_nerfs_b200.mesh import Mesh, write_ply
    z = torch.zeros(0, 3)
    path = str(tmp_path / "e.ply")
    write_ply(path, Mesh(z, z, z, torch.zeros(0, 3, dtype=torch.int32)))
    rv, _, _, rf = M.read_ply(path)
    assert rv.shape == (0, 3) and rf.shape == (0, 3)


# ---- flags -------------------------------------------------------------------------------------------------------
def test_mesh_flags():
    from opt import get_opts
    h = get_opts([])
    assert (h.extract_mesh, h.mesh_res, h.mesh_threshold, h.mesh_bound) == (False, 512, 10.0, 0.0)
    h = get_opts(["--extract_mesh", "--mesh_res", "2", "--mesh_bound", "0.5", "--mesh_threshold", "-3"])
    assert h.extract_mesh and h.mesh_res == 2 and h.mesh_bound == 0.5
    assert get_opts(["--mesh_res", "1024", "--scale", "2", "--mesh_bound", "1.5"]).mesh_res == 1024


@pytest.mark.parametrize("args", [["--mesh_res", "1"], ["--mesh_res", "1025"], ["--mesh_threshold", "nan"],
                                  ["--mesh_threshold", "inf"], ["--mesh_bound", "-0.1"], ["--mesh_bound", "0.6"],
                                  ["--mesh_bound", "nan"], ["--scale", "2", "--mesh_bound", "2.5"]])
def test_mesh_flags_rejected(args):
    from opt import get_opts
    with pytest.raises(SystemExit):
        get_opts(args)


# ---- C-ABI -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def test_mesh_argument_validation_needs_no_gpu(lib):
    nan, inf = float("nan"), float("inf")
    assert lib.ngp_mc_workspace_bytes(1) < 0 and lib.ngp_mc_workspace_bytes(1025) < 0
    assert lib.ngp_mc_workspace_bytes(2) > 0 and lib.ngp_mc_workspace_bytes(1024) > lib.ngp_mc_workspace_bytes(512)
    assert lib.ngp_mc_count(None, 1, 0.0, None, None) < 0
    assert lib.ngp_mc_count(None, 64, nan, None, None) < 0
    assert b"finite" in lib.ngp_last_error()
    assert lib.ngp_mc_count(None, 64, inf, None, None) < 0
    assert lib.ngp_mc_count(None, 64, 0.0, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert lib.ngp_mc_scan(2000, None, None, None) < 0
    assert lib.ngp_mc_scan(64, None, None, None) < 0
    assert lib.ngp_mc_emit_vertices(None, 64, 0.0, 1.0, None, 1 << 31, None, None, None, None) < 0
    assert b"2^31" in lib.ngp_last_error()
    assert lib.ngp_mc_emit_vertices(None, 64, 0.0, 0.0, None, 5, None, None, None, None) < 0
    assert lib.ngp_mc_emit_faces(None, 64, 0.0, None, None, 1 << 31, None, None) < 0
    assert lib.ngp_mc_emit_faces(None, 64, 0.0, None, None, -1, None, None) < 0
    assert lib.ngp_mesh_lattice_points(1, 0.5, 0, 8, None, 1, 128, 0.5, None, None, None) < 0
    assert lib.ngp_mesh_lattice_points(8, 0.6, 0, 8, None, 1, 128, 0.5, None, None, None) < 0
    assert b"bound" in lib.ngp_last_error()
    assert lib.ngp_mesh_lattice_points(8, 0.5, 500, 13, None, 1, 128, 0.5, None, None, None) < 0
    assert lib.ngp_mesh_lattice_points(8, 0.5, 0, 8, None, 1, 128, 0.5, None, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert lib.ngp_mesh_lattice_store(None, None, -1, 8, None, None) < 0
    assert lib.ngp_mesh_lattice_store(None, None, 0, 8, None, None) < 0
    # empty ranges are a no-op success
    assert lib.ngp_mesh_lattice_points(8, 0.5, 0, 0, None, 1, 128, 0.5, None, None, None) == 0
    assert lib.ngp_mesh_lattice_store(None, None, 0, 0, None, None) == 0
    assert lib.ngp_mc_emit_vertices(C.c_void_p(1), 64, 0.0, 1.0, C.c_void_p(1), 0, C.c_void_p(1), None, None,
                                     None) == 0
