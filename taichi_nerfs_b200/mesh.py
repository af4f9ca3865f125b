"""Mesh export of a trained model (DESIGN.md §6g): the density lattice, marching cubes on the device, vertex colours
from the model's own forward, and a binary PLY writer.

    mesh = extract_mesh(model, 512, 10.0)
    write_ply('results/mesh.ply', mesh)

Works for every model kind: NGP with the hash (fp32 or --half_opt) or tri-plane encoder, the --deployment
architecture, and the voxel grid.  Surfaces that reach the lattice border stay open: the lattice is not padded.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

from . import ops

LATTICE_CHUNK = 1 << 21       # nodes per density evaluation: bounds the encoder's embedding buffers
COLOR_CHUNK = 1 << 20         # vertices per colour evaluation


class Mesh(NamedTuple):
    vertices: torch.Tensor    # [V, 3] fp32 world positions
    normals: torch.Tensor     # [V, 3] fp32 unit, outward (toward lower density)
    colors: torch.Tensor      # [V, 3] fp32 rgb in [0, 1], seen along -normal
    faces: torch.Tensor       # [F, 3] int32, counter-clockwise seen from outside


def _bound(model, bound):
    scale = float(model.scale)
    b = scale if bound is None or bound == 0 else float(bound)
    if not (math.isfinite(b) and 0 < b <= scale):
        raise ValueError(f"mesh bound must lie in (0, scale = {scale}], got {bound}")
    return b


@torch.no_grad()
def density_lattice(model, n, bound=None):
    """fp32 [n, n, n] lattice of the model's density over [-bound, bound]^3 (bound defaults to model.scale): sigma where
    the node lies in an occupied cell of the model's occupancy grid and sigma is finite, 0 elsewhere."""
    n = int(n)
    if not 2 <= n <= 1024:
        raise ValueError(f"lattice size must be in [2, 1024], got {n}")
    b = _bound(model, bound)
    bits = model.density_bitfield
    lattice = torch.empty(n, n, n, device=bits.device, dtype=torch.float32)
    total = n ** 3
    for start in range(0, total, LATTICE_CHUNK):
        count = min(LATTICE_CHUNK, total - start)
        xyz, occ = ops.mesh_lattice_points(n, b, start, count, bits, model.cascades, model.grid_size, model.scale)
        with torch.autocast(device_type='cuda', dtype=torch.float16):   # the density path of the grid update
            sigma = model._density_eval(xyz)
        ops.mesh_lattice_store(sigma.float(), occ, start, lattice)
    return lattice


@torch.no_grad()
def vertex_colors(model, vertices, normals):
    """rgb [V, 3] fp32 of the model at each vertex, seen along d = -normal (a camera outside looking at the surface)."""
    out = torch.empty_like(vertices)
    for i in range(0, len(vertices), COLOR_CHUNK):
        x = vertices[i:i + COLOR_CHUNK].contiguous()
        d = (-normals[i:i + COLOR_CHUNK]).contiguous()
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            _, rgb = model(x, d)
        out[i:i + COLOR_CHUNK] = rgb.float()
    return out


@torch.no_grad()
def extract_mesh(model, n, threshold, bound=None):
    """Marching cubes of ``density_lattice(model, n, bound)`` at ``threshold``, with the model's colours: a ``Mesh``
    on the model's device."""
    if not math.isfinite(threshold):
        raise ValueError(f"mesh threshold must be finite, got {threshold}")
    b = _bound(model, bound)
    lattice = density_lattice(model, n, b)
    vertices, normals, faces = ops.marching_cubes(lattice, threshold, b)
    del lattice
    return Mesh(vertices, normals, vertex_colors(model, vertices, normals), faces)


PLY_VERTEX = np.dtype([('x', '<f4'), ('y', '<f4'), ('z', '<f4'), ('nx', '<f4'), ('ny', '<f4'), ('nz', '<f4'),
                       ('red', 'u1'), ('green', 'u1'), ('blue', 'u1')])
PLY_FACE = np.dtype([('n', 'u1'), ('i', '<u4', (3,))])


def write_ply(path, mesh):
    """Binary little-endian PLY: per vertex float x y z, float nx ny nz, uchar red green blue; faces as
    list uchar uint32 vertex_indices.  Colours are rounded from [0, 1] to 0..255."""
    v = mesh.vertices.detach().float().cpu().numpy().reshape(-1, 3)
    nrm = mesh.normals.detach().float().cpu().numpy().reshape(-1, 3)
    rgb = mesh.colors.detach().float().clamp(0, 1).cpu().numpy().reshape(-1, 3)
    f = mesh.faces.detach().cpu().numpy().reshape(-1, 3)
    verts = np.empty(len(v), PLY_VERTEX)
    for k, name in enumerate(('x', 'y', 'z')):
        verts[name] = v[:, k]
    for k, name in enumerate(('nx', 'ny', 'nz')):
        verts[name] = nrm[:, k]
    rgb8 = np.rint(rgb * 255.0).astype(np.uint8)
    for k, name in enumerate(('red', 'green', 'blue')):
        verts[name] = rgb8[:, k]
    faces = np.empty(len(f), PLY_FACE)
    faces['n'] = 3
    faces['i'] = f.astype(np.uint32)
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(verts)}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property float nx\nproperty float ny\nproperty float nz\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {len(faces)}\n"
              "property list uchar uint32 vertex_indices\n"
              "end_header\n")
    with open(path, 'wb') as fh:
        fh.write(header.encode('ascii'))
        fh.write(verts.tobytes())
        fh.write(faces.tobytes())
