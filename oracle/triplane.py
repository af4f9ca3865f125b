"""ctypes/numpy binding of the tri-plane CPU oracle (oracle/triplane.c) and the oracle training step / frame of a
tri-plane model — TEST INFRASTRUCTURE ONLY (tests/), never imported by the product packages.

The step and frame follow oracle/train_step.py (train.py:168-201, modules/rendering.py:61-228) with the hash encoder
replaced by the tri-plane encoder (modules/networks.py:101-107: fp32 plane table, no fp16 shadow); everything else is
the oracle's own kernels.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import oracle as O
from .train_step import OracleModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "triplane.c")
_SO = os.path.join(_HERE, "build", "libtriplane_oracle.so")
# the flags of oracle/Makefile: strict fp32, no mul+add contraction
CFLAGS = ["-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-Wall", "-Wextra", "-std=gnu11"]


def build(force: bool = False) -> str:
    hdr = os.path.join(_HERE, "..", "include", "ngp_b200.h")
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in (_SRC, hdr))
    if force or stale:
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.run([cc] + CFLAGS + ["-shared", "-o", _SO, _SRC, "-lm"], check=True)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
    return _lib


def triplane_encode_fwd(xyz, table, layout):
    """Tri-plane encoder forward (modules/triplane.py:35-98), xyz [n,3] in [0,1] -> fp32 [n, L*F] (feature-major)."""
    x = O._c(xyz, np.float32)
    tab = O._c(table, np.float32)
    n = x.shape[0]
    out = np.empty((n, layout.out_dim), np.float32)
    cl = layout.as_ctypes()
    O._chk(lib().ngp_triplane_encode_fwd_cpu(O._p(x), O._p(tab), C.byref(cl), O._p(out), C.c_int64(n)))
    return out


def triplane_encode_bwd(xyz, table, dout, layout, grad_table=None):
    """Gradient of sum(dout * fwd) wrt the plane table (Taichi autodiff, triplane.py:186-197), accumulated into
    grad_table (fp32 [P], zeros when None)."""
    x = O._c(xyz, np.float32)
    tab, dy = O._c(table, np.float32), O._c(dout, np.float32)
    if grad_table is None:
        grad_table = np.zeros(layout.total_param_size, np.float32)
    cl = layout.as_ctypes()
    O._chk(lib().ngp_triplane_encode_bwd_cpu(O._p(x), O._p(tab), O._p(dy), C.byref(cl), O._p(grad_table),
                                             C.c_int64(x.shape[0])))
    return grad_table


class TriplaneOracleModel(OracleModel):
    """OracleModel of a tri-plane NGP: ``layout`` is a TriplaneLayout, ``table`` the flat fp32 plane table."""

    def __init__(self, layout, table, mlp_weights, bitfield, scale=0.5, cascades=1, grid_size=128):
        super().__init__(layout, table, mlp_weights, bitfield, scale, cascades, grid_size, half=False)


def _normalise(model, xyzs):
    lo, hi = np.float32(-model.scale), np.float32(model.scale)   # networks.py:144
    return ((xyzs - lo) / (hi - lo)).astype(np.float32)


def forward(model, rays_o, rays_d, noise, exp_step_factor=0.0, T_threshold=1e-4, max_samples=1024):
    """train_step.forward with the tri-plane encoder."""
    hits = O.ray_aabb_intersect(rays_o, rays_d, model.scale)
    rays_a, xyzs, dirs, deltas, ts, S = O.raymarching_train(rays_o, rays_d, hits, model.bitfield, noise,
                                                           model.cascades, model.scale, exp_step_factor,
                                                           model.grid_size, max_samples)
    xn = _normalise(model, xyzs)
    emb = triplane_encode_fwd(xn, model.table, model.layout)
    sigmas, rgbs = O.mlp_fwd(emb, dirs, model.ws)
    tot, opacity, depth, rgb, ws = O.composite_train_fwd(sigmas, rgbs, deltas, ts, rays_a, T_threshold)
    bg = np.float32(1.0 if exp_step_factor == 0 else 0.0)  # rendering.py:219-226
    rgb_out = rgb + bg * (1 - opacity)[:, None]
    cache = dict(hits=hits, rays_a=rays_a, xn=xn, dirs=dirs, deltas=deltas, ts=ts, emb=emb, sigmas=sigmas,
                 rgbs=rgbs, opacity=opacity, rgb=rgb, bg=bg, S=S, vr_samples=int(tot.sum()), T_threshold=T_threshold)
    return rgb_out.astype(np.float32), cache


def render_test(model, rays_o, rays_d, exp_step_factor=0.0, T_threshold=1e-4, max_samples=1024):
    """train_step.render_test with the tri-plane encoder (same returned dict)."""
    n = rays_o.shape[0]
    hits = O.ray_aabb_intersect(rays_o, rays_d, model.scale)
    rays_a, xyzs, dirs, deltas, ts, S = O.raymarching_train(rays_o, rays_d, hits, model.bitfield,
                                                           np.zeros(n, np.float32), model.cascades, model.scale,
                                                           exp_step_factor, model.grid_size, max_samples)
    emb = triplane_encode_fwd(_normalise(model, xyzs), model.table, model.layout)
    sigmas, rgbs = O.mlp_fwd(emb, dirs, model.ws)
    opacity, depth = np.zeros(n, np.float32), np.zeros(n, np.float32)
    rgb = np.zeros((n, 3), np.float32)
    O.composite_test(sigmas, rgbs, deltas, ts, rays_a[:, 1:].astype(np.int64), rays_a[:, 0].astype(np.int64),
                     T_threshold, opacity, depth, rgb)
    n_term = O.composite_train_fwd(sigmas, rgbs, deltas, ts, rays_a, T_threshold)[0]
    bg = np.float32(1.0 if exp_step_factor == 0 else 0.0)  # rendering.py:152-156
    return dict(rgb=(rgb + bg * (1 - opacity)[:, None]).astype(np.float32), depth=depth, opacity=opacity, S=S,
                n_term=n_term, rays_a=rays_a, sigmas=sigmas, deltas=deltas)


def backward(model, cache, rgb_out, rgb_gt, loss_scale):
    """train_step.backward with the tri-plane encoder: (loss, grad_table fp32 [P], grad_mlp fp32 [9408]) of
    loss*loss_scale."""
    n = rgb_out.shape[0]
    diff = rgb_out - rgb_gt
    loss = float((diff.astype(np.float64) ** 2).mean())
    g_rgb = (np.float32(loss_scale) * 2.0 * diff / np.float32(3 * n)).astype(np.float32)
    g_op = (-cache['bg'] * g_rgb.sum(1)).astype(np.float32)
    S = cache['S']
    dsig, drgbs = O.composite_train_bwd(g_op, np.zeros(n, np.float32), g_rgb, np.zeros(S, np.float32),
                                        cache['sigmas'], cache['rgbs'], cache['deltas'], cache['ts'],
                                        cache['rays_a'], cache['T_threshold'])
    demb, g_mlp = O.mlp_bwd(cache['emb'], cache['dirs'], model.ws, dsig, drgbs)
    g_table = triplane_encode_bwd(cache['xn'], model.table, demb, model.layout)
    return loss, g_table, g_mlp
