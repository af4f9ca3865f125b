"""CPU restatement of ONE full training step of the reference (train.py:168-201) composed from the
oracle kernels — TEST INFRASTRUCTURE (tests/, smoke(), bench.py cpu_baseline / --impl reference only).

Follows, in order: datasets/ray_utils.py:51-80 (get_rays), modules/rendering.py:12-57,161-228
(render/train path), modules/networks.py:136-166 (NGP.forward), torch.nn.functional.mse_loss,
the Taichi autodiff / hand-written backward kernels cited in ngp_oracle.c, and
GradScaler + torch.optim.Adam(eps=1e-15) (train.py:137-156,197-201).
"""
from __future__ import annotations

import numpy as np

from . import oracle as O


def make_rays(n, seed=0, radius=1.4, img=800, focal=1111.111, img_h=None):
    """Lego-shape synthetic rays (numpy): pinhole 800x800 fx=fy=1111.111 (datasets/nsvf.py:37-44), cameras on
    the upper hemisphere looking at the origin, [right, down, front] convention (datasets/ray_utils.py:8-80).
    ``img`` x ``img_h`` (default square) pixels."""
    rng = np.random.default_rng(seed)
    th = rng.uniform(0, 2 * np.pi, n)
    ph = np.arccos(rng.uniform(0.05, 0.95, n))
    c = np.stack([np.sin(ph) * np.cos(th), np.sin(ph) * np.sin(th), np.cos(ph)], -1) * radius
    fwd = -c / np.linalg.norm(c, axis=-1, keepdims=True)
    right = np.cross(fwd, np.array([0, 0, 1.0]))
    right /= np.linalg.norm(right, axis=-1, keepdims=True)
    down = np.cross(fwd, right)
    img_h = img if img_h is None else img_h
    u = rng.integers(0, img, n)
    v = rng.integers(0, img_h, n)
    dc = np.stack([(u - img / 2 + .5) / focal, (v - img_h / 2 + .5) / focal, np.ones(n)], -1)
    d = dc[:, 0:1] * right + dc[:, 1:2] * down + dc[:, 2:3] * fwd
    return c.astype(np.float32), d.astype(np.float32)


class OracleModel:
    """Plain-numpy parameter container mirroring NGP's state (half_opt: fp32 master [entries,2] +
    fp16 shadow; fp32 mode: flat fp32 table)."""

    def __init__(self, layout, table, mlp_weights, bitfield, scale=0.5, cascades=1, grid_size=128, half=True):
        self.layout = layout
        self.table = np.ascontiguousarray(table, np.float32).reshape(-1)
        self.ws = [np.ascontiguousarray(w, np.float32) for w in mlp_weights]
        self.bitfield = np.ascontiguousarray(bitfield, np.uint8)
        self.scale, self.cascades, self.grid_size, self.half = float(scale), int(cascades), int(grid_size), bool(half)
        self.shadow = self.table.astype(np.float16) if half else None
        n = self.table.size + sum(w.size for w in self.ws)
        self.m = np.zeros(n, np.float32)
        self.v = np.zeros(n, np.float32)
        self.step = 0

    def table_for_kernel(self):
        return self.shadow if self.half else self.table


def forward(model, rays_o, rays_d, noise, exp_step_factor=0.0, T_threshold=1e-4, max_samples=1024):
    hits = O.ray_aabb_intersect(rays_o, rays_d, model.scale)
    rays_a, xyzs, dirs, deltas, ts, S = O.raymarching_train(rays_o, rays_d, hits, model.bitfield, noise,
                                                           model.cascades, model.scale, exp_step_factor,
                                                           model.grid_size, max_samples)
    # NGP.density: x = (x - xyz_min) / (xyz_max - xyz_min), fp32 (networks.py:144)
    lo, hi = np.float32(-model.scale), np.float32(model.scale)
    xn = ((xyzs - lo) / (hi - lo)).astype(np.float32)
    emb = O.hash_encode_fwd(xn, model.table_for_kernel(), model.layout)
    sigmas, rgbs = O.mlp_fwd(emb, dirs, model.ws)
    tot, opacity, depth, rgb, ws = O.composite_train_fwd(sigmas, rgbs, deltas, ts, rays_a, T_threshold)
    bg = np.float32(1.0 if exp_step_factor == 0 else 0.0)  # rendering.py:219-226
    rgb_out = rgb + bg * (1 - opacity)[:, None]
    cache = dict(hits=hits, rays_a=rays_a, xn=xn, dirs=dirs, deltas=deltas, ts=ts, emb=emb, sigmas=sigmas,
                 rgbs=rgbs, opacity=opacity, rgb=rgb, bg=bg, S=S, vr_samples=int(tot.sum()), T_threshold=T_threshold)
    return rgb_out.astype(np.float32), cache


def render_test(model, rays_o, rays_d, exp_step_factor=0.0, T_threshold=1e-4, max_samples=1024):
    """render(test_time=True) of the reference (modules/rendering.py:61-158) in one pass: the test-time march (no
    jitter, at most max_samples per ray) of every ray, the network on every sample, then ONE composite_test call over
    each ray's whole sample list.  Compositing stops at the first sample where T <= T_threshold, so this equals the
    reference's chunked loop whenever that loop does not stop a ray early at max_samples (tests/test_oracle.py).
    Returns dict(rgb [N,3] background included, depth [N], opacity [N], S = samples marched, n_term [N] = samples per
    ray up to and including the one where T falls to the threshold, rays_a, sigmas, deltas)."""
    n = rays_o.shape[0]
    hits = O.ray_aabb_intersect(rays_o, rays_d, model.scale)
    rays_a, xyzs, dirs, deltas, ts, S = O.raymarching_train(rays_o, rays_d, hits, model.bitfield,
                                                           np.zeros(n, np.float32), model.cascades, model.scale,
                                                           exp_step_factor, model.grid_size, max_samples)
    lo, hi = np.float32(-model.scale), np.float32(model.scale)
    xn = ((xyzs - lo) / (hi - lo)).astype(np.float32)
    sigmas, rgbs = O.mlp_fwd(O.hash_encode_fwd(xn, model.table_for_kernel(), model.layout), dirs, model.ws)
    opacity, depth = np.zeros(n, np.float32), np.zeros(n, np.float32)
    rgb = np.zeros((n, 3), np.float32)
    O.composite_test(sigmas, rgbs, deltas, ts, rays_a[:, 1:].astype(np.int64), rays_a[:, 0].astype(np.int64),
                     T_threshold, opacity, depth, rgb)
    n_term = O.composite_train_fwd(sigmas, rgbs, deltas, ts, rays_a, T_threshold)[0]  # same loop, counts the samples
    bg = np.float32(1.0 if exp_step_factor == 0 else 0.0)  # rendering.py:152-156
    return dict(rgb=(rgb + bg * (1 - opacity)[:, None]).astype(np.float32), depth=depth, opacity=opacity, S=S,
                n_term=n_term, rays_a=rays_a, sigmas=sigmas, deltas=deltas)


def backward(model, cache, rgb_out, rgb_gt, loss_scale):
    """Returns (loss, grad_table fp32 [P], grad_mlp fp32 [9408]) — gradients of loss*loss_scale."""
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
    g_table = O.hash_encode_bwd(cache['xn'], demb, model.layout)
    return loss, g_table, g_mlp


def adam(model, g_table, g_mlp, lr, loss_scale, world_size=1):
    model.step += 1
    inv = 1.0 / (loss_scale * world_size)
    if O.check_finite(g_table) or O.check_finite(g_mlp):
        return False
    P = model.table.size
    O.adam_step(model.table, g_table, model.m[:P], model.v[:P], lr, model.step, inv_scale=inv,
                param_f16=model.shadow)
    off = P
    goff = 0
    for w in model.ws:
        flat = w.reshape(-1)
        g = np.ascontiguousarray(g_mlp[goff:goff + flat.size])
        O.adam_step(flat, g, model.m[off:off + flat.size], model.v[off:off + flat.size], lr, model.step, inv_scale=inv)
        off += flat.size
        goff += flat.size
    return True


def train_step(model, rays_o, rays_d, rgb_gt, noise, lr=1e-2, loss_scale=65536.0, exp_step_factor=0.0):
    rgb_out, cache = forward(model, rays_o, rays_d, noise, exp_step_factor)
    loss, g_table, g_mlp = backward(model, cache, rgb_out, rgb_gt, loss_scale)
    adam(model, g_table, g_mlp, lr, loss_scale)
    return loss, cache
