"""Test-time frame rendering without the host-driven while-loop.

The reference renders a frame (gui.py:115-145 -> modules/rendering.py:61-158) by repeatedly marching
<= N samples per alive ray, compacting with boolean masks (host syncs), running the network and
compositing incrementally, until every ray has terminated — hundreds of tiny launches and >= 3 host
syncs per iteration.  Compositing is sequential per ray and stops at the first sample where the
transmittance falls to <= T_threshold, so the result does not depend on how the samples are chunked.
Here the frame is rendered in a few big launches per ray block: march ALL samples of the block
(warp-per-ray march, deterministic layout), encode + MLP them in one pass each, composite with the
warp-per-ray kernel that applies the same early termination.  Samples behind an opaque surface are
evaluated but ignored (the price of no per-iteration sync); the rendered rgb/depth/opacity equal the
loop's up to fp rounding.
"""
from __future__ import annotations

import torch

from . import ops
from .fused_mlp import mlp_weights


@torch.no_grad()
def render_frame(model, rays_o, rays_d, exp_step_factor=0.0, T_threshold=1e-4, max_samples=1024,
                 block_rays=1 << 18):
    """Returns the dict of rendering.render(test_time=True): rgb [N,3], depth [N], opacity [N], total_samples."""
    dev = rays_o.device
    n = rays_o.shape[0]
    rays_o = rays_o.float().contiguous()
    rays_d = rays_d.float().contiguous()
    rgb = torch.empty(n, 3, device=dev, dtype=torch.float32)
    depth = torch.empty(n, device=dev, dtype=torch.float32)
    opacity = torch.empty(n, device=dev, dtype=torch.float32)
    enc = model.pos_encoder
    fused = bool(model._fusable(rays_o))     # stock architecture: encoder + fused MLP kernels on the raw sample rows
    if fused:
        W = [w.detach() for w in mlp_weights(model)]
    aabb = model.xyz_min.flatten().tolist() + (model.xyz_max - model.xyz_min).flatten().tolist()
    total = 0
    zeros = torch.zeros(min(block_rays, n), device=dev, dtype=torch.float32)  # test-time march has no jitter
    caps = model.__dict__.setdefault('_frame_capacity', {})  # learned per ray block from the previous frame
    for b in range(0, n, block_rays):
        e = min(b + block_rays, n)
        o, d = rays_o[b:e], rays_d[b:e]
        hits = ops.ray_aabb_intersect(o, d, model.scale)
        key = (b, e - b)
        done = False
        if key in caps and max_samples <= 1024:
            # single-pass march: each ray reserves its rows with one atomic; capacity from the last frame
            cap = caps[key]
            counter = torch.zeros(2, device=dev, dtype=torch.int32)
            rays_a = torch.empty(e - b, 3, device=dev, dtype=torch.int32)
            xyzs = torch.empty(cap, 3, device=dev, dtype=torch.float32)
            dirs = torch.empty(cap, 3, device=dev, dtype=torch.float32)
            deltas = torch.empty(cap, device=dev, dtype=torch.float32)
            ts = torch.empty(cap, device=dev, dtype=torch.float32)
            ops.raymarching_frame(o, d, hits, model.density_bitfield, model.cascades, model.scale, exp_step_factor,
                                  model.grid_size, max_samples, counter, rays_a, xyzs, dirs, deltas, ts)
            S, dropped = counter.tolist()  # one host read per ray block
            caps[key] = max(int(S * 1.25) + 4096, 1 << 16)
            if dropped == 0:
                done = True
                xyzs, dirs, deltas, ts = xyzs[:S], dirs[:S], deltas[:S], ts[:S]
        if not done:
            # exact two-pass march (count -> scan -> write); also used for the first frame to learn S
            noise = zeros[: e - b]
            counter, rays_a = ops.raymarching_train_count(o, d, hits, model.density_bitfield, noise, model.cascades,
                                                          model.scale, exp_step_factor, model.grid_size, max_samples)
            S = int(counter[0].item())
            caps[key] = max(int(S * 1.25) + 4096, 1 << 16)
            if S > 0:
                xyzs = torch.empty(S, 3, device=dev, dtype=torch.float32)
                dirs = torch.empty(S, 3, device=dev, dtype=torch.float32)
                deltas = torch.empty(S, device=dev, dtype=torch.float32)
                ts = torch.empty(S, device=dev, dtype=torch.float32)
                ops.raymarching_train_write(o, d, hits, model.density_bitfield, noise, model.cascades, model.scale,
                                            exp_step_factor, model.grid_size, counter, rays_a, xyzs, dirs, deltas, ts)
        total += S
        if S == 0:
            opacity[b:e] = 0
            depth[b:e] = 0
            rgb[b:e] = 0
            continue
        if fused:
            emb = enc.encode_world(xyzs, aabb)  # hash or tri-plane kernel, normalisation in-kernel
            sigmas, rgbs = ops.mlp_fwd(emb, dirs, W)
        else:   # any other NGP configuration (e.g. the reference's L=4 F=4 deployment model): module forward
            with torch.autocast('cuda', dtype=torch.float16):
                outs = [model(xyzs[i:i + (1 << 21)], dirs[i:i + (1 << 21)]) for i in range(0, S, 1 << 21)]
            sigmas = torch.cat([o[0] for o in outs]).float().contiguous()
            rgbs = torch.cat([o[1] for o in outs]).contiguous()
        _, op_b, dp_b, rgb_b, _ = ops.composite_train_fwd(sigmas, rgbs, deltas, ts, rays_a, T_threshold)
        opacity[b:e] = op_b
        depth[b:e] = dp_b
        rgb[b:e] = rgb_b
    bg = 1.0 if exp_step_factor == 0 else 0.0  # rendering.py:152-156
    if bg:
        rgb += bg * (1 - opacity)[:, None]
    return {'opacity': opacity, 'depth': depth, 'rgb': rgb, 'total_samples': torch.tensor(total, device=dev)}


# =====================================================================================================
class FrameRenderer:
    """Compacting test-time renderer: the whole frame is ONE CUDA graph of rounds with device-side control.

    round = [bookkeeping] -> persistent-warp march over the list of live rays (<= limit samples per ray, resume point
    kept per ray) -> hash encode -> fused MLP -> composite onto the per-ray accumulators + block-level compaction of
    the rays that are still alive (transmittance above the threshold, still inside the box) into the next round's list.
    Rays that have hit an opaque surface leave the list, so — unlike ``render_frame`` — samples behind it are neither
    marched nor shaded.  The host reads nothing until the frame is done (one 32-byte state read), where the reference
    synchronises several times per iteration (modules/rendering.py:96-144).  The per-ray result equals the loop's up to
    fp rounding: compositing is sequential per ray and stops at the first sample with T <= threshold, however the
    samples are grouped into rounds.
    """
    SCHEDULE = (4, 8, 16, 32, 64, 128, 256, 512, 4)     # samples per live ray and round; sums to max_samples = 1024
    MAX_SAMPLES = 1024     # per ray over the whole frame, extra rounds included (the one-shot march's max_samples)

    def __init__(self, model, n_rays, exp_step_factor=0.0, T_threshold=1e-4, rows_per_ray=6, use_graph=True,
                 use_leap=True):
        import ctypes as C
        from ._lib import F16, F32, MlpWeights, check, load
        self._C, self._check, self._load = C, check, load
        self.model = model
        dev = model.density_bitfield.device
        enc = model.pos_encoder
        self.dev, self.n = dev, int(n_rays)
        self.cap = int(n_rays) * int(rows_per_ray)
        self.esf, self.T_thr = float(exp_step_factor), float(T_threshold)
        edt = enc.emb_dtype     # fp16 (half_opt hash) or fp32 (fp32 hash, tri-plane) embedding
        self.tag = F16 if edt == torch.float16 else F32
        f32, i32 = torch.float32, torch.int32
        z = lambda *s, dtype=f32: torch.zeros(*s, device=dev, dtype=dtype)  # noqa: E731
        n, cap = self.n, self.cap
        self.rays_o, self.rays_d, self.hits = z(n, 3), z(n, 3), z(n, 2)
        self.t_cur, self.state = z(n), z(8, dtype=i32)
        self.n_marched = z(n, dtype=i32)         # per ray: samples marched so far in this frame (capped at MAX_SAMPLES)
        self.alive = [z(n, dtype=i32), z(n, dtype=i32)]
        self.rays_a = z(n, 3, dtype=i32)
        self.xyzs, self.dirs, self.deltas, self.ts = z(cap, 3), z(cap, 3), z(cap), z(cap)
        self.emb, self.sig, self.rgbs = z(cap, 32, dtype=edt), z(cap), z(cap, 3, dtype=torch.float16)
        self.opacity, self.depth, self.rgb = z(n), z(n), z(n, 3)
        self.coarse = None
        import os
        # The empty-space leap of the round march is opt-in (NGP_FRAME_LEAP=1): bit-exact (tests), but its exact
        # super-cell box test cost more than the steps it skips on the Lego-sized box when it was measured.
        use_leap = use_leap and os.environ.get("NGP_FRAME_LEAP", "0") == "1"
        if use_leap and model.cascades == 1 and model.grid_size in (32, 64, 128) and self.esf == 0.0:
            self.coarse = z(max((model.grid_size // 8) ** 3 // 32, 1), dtype=i32)
        self.aabb6 = (C.c_float * 6)(*[float(v) for v in model.xyz_min.flatten().tolist()],
                                     *[float(v) for v in (model.xyz_max - model.xyz_min).flatten().tolist()])
        self._w_keep = [w.detach().float().contiguous() for w in mlp_weights(model)]
        self._wst = MlpWeights(*[w.data_ptr() for w in self._w_keep])
        self._w_ptrs = [w.data_ptr() for w in mlp_weights(model)]
        self.rays_o[:] = torch.tensor([1.2, 0.3, 0.5], device=dev)      # valid placeholder rays for the capture
        self.rays_d[:] = -self.rays_o
        self.graph = None
        self.rounds_run = 0
        if use_graph:
            self._capture()

    def _p(self, t):
        return None if t is None else self._C.c_void_p(t.data_ptr())

    def _table(self):
        return self.model.pos_encoder.kernel_table()

    def _enqueue_round(self, j, limit):
        L, m, st, p, check = self._load(), self.model, self._C.c_void_p(torch.cuda.current_stream().cuda_stream), self._p, self._check
        cur, nxt = self.alive[j & 1], self.alive[(j + 1) & 1]
        check(L.ngp_frame_round_begin(p(self.state), st))
        check(L.ngp_raymarching_round_capped(p(self.rays_o), p(self.rays_d), p(self.hits), p(m.density_bitfield),
                                             m.cascades, m.grid_size, float(m.scale), self.esf, int(limit),
                                             self.MAX_SAMPLES, p(cur), p(self.state), p(self.t_cur), p(self.n_marched),
                                             p(self.rays_a), p(self.xyzs), p(self.dirs), p(self.deltas), p(self.ts),
                                             self.n, self.cap, p(self.coarse), st))
        check(m.pos_encoder.enqueue_encode_dyn(L, p(self.xyzs), p(self._table_t), p(self.emb), self.cap, p(self.state),
                                               self.aabb6, st))
        check(L.ngp_mlp_fwd_dyn(p(self.emb), self.tag, p(self.dirs), self._C.byref(self._wst), p(self.sig), p(self.rgbs),
                                None, self.cap, p(self.state), st))
        check(L.ngp_composite_round(p(self.sig), p(self.rgbs), 1, p(self.deltas), p(self.ts), p(self.rays_a),
                                    p(self.state), p(self.t_cur), p(self.hits), self.T_thr, p(self.opacity),
                                    p(self.depth), p(self.rgb), p(nxt), self.n, int(limit), st))

    def _enqueue_frame(self):
        L, m, st, p, check = self._load(), self.model, self._C.c_void_p(torch.cuda.current_stream().cuda_stream), self._p, self._check
        check(L.ngp_ray_aabb_intersect(p(self.rays_o), p(self.rays_d), float(m.scale), p(self.hits), self.n, st))
        check(L.ngp_frame_begin(p(self.hits), p(self.t_cur), p(self.n_marched), p(self.alive[0]), p(self.state),
                                p(self.opacity), p(self.depth), p(self.rgb), self.n, st))
        if self.coarse is not None:   # 8^3-cell dilated occupancy: lets the march leap over empty space
            check(L.ngp_build_coarse_occupancy(p(m.density_bitfield), m.grid_size, p(self.coarse), st))
        for j, limit in enumerate(self.SCHEDULE):
            self._enqueue_round(j, limit)

    def _capture(self):
        self._table_t = self._table()
        self._table_ptr = self._table_t.data_ptr()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._enqueue_frame()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._enqueue_frame()

    @torch.no_grad()
    def render(self, rays_o, rays_d):
        """-> the dict of rendering.render(test_time=True).  Output tensors are views of static buffers (valid until
        the next call)."""
        self.rays_o.copy_(rays_o, non_blocking=True)
        self.rays_d.copy_(rays_d, non_blocking=True)
        tab = self._table()
        if self.graph is not None and tab.data_ptr() == self._table_ptr:
            self.graph.replay()
        else:   # eager enqueue (no graph, or the table the encoder reads was re-allocated since the capture)
            self._table_t = tab
            self._enqueue_frame()
        rounds = len(self.SCHEDULE)
        # the one host read of the frame: state = [rows of the last round, -, live rays of the last round,
        # live rays left for a further round, samples evaluated before the last round, ...]
        st = self.state.tolist()
        j = rounds
        while st[3] > 0:   # rays that need more than the scheduled rounds (un-trained / foggy models), up to MAX_SAMPLES
            self._table_t = tab
            self._enqueue_round(j, 512)
            st = self.state.tolist()
            j += 1
            if j > rounds + 4096:
                raise RuntimeError("FrameRenderer: rays never terminate")
        self.rounds_run = j
        bg = 1.0 if self.esf == 0 else 0.0     # rendering.py:152-156
        rgb = self.rgb + bg * (1 - self.opacity)[:, None] if bg else self.rgb.clone()
        # results are copies: the static buffers are overwritten by the next frame
        return {'opacity': self.opacity.clone(), 'depth': self.depth.clone(), 'rgb': rgb,
                'total_samples': torch.tensor(st[4] + st[0], device=self.dev)}


def render_frame_compact(model, rays_o, rays_d, exp_step_factor=0.0, T_threshold=1e-4, max_samples=1024):
    """render(test_time=True) through a cached FrameRenderer (one per model, ray count and render settings)."""
    if max_samples != 1024:
        return render_frame(model, rays_o, rays_d, exp_step_factor, T_threshold, max_samples)
    cache = model.__dict__.setdefault('_frame_renderers', {})
    key = (rays_o.shape[0], float(exp_step_factor), float(T_threshold), rays_o.device)
    fr = cache.get(key)
    if fr is not None and [w.data_ptr() for w in mlp_weights(model)] != fr._w_ptrs:
        fr = None       # parameters were re-bound (e.g. an NGPTrainer adopted them): the captured pointers are stale
    if fr is None:
        if len(cache) >= 2:
            cache.clear()
        fr = cache[key] = FrameRenderer(model, rays_o.shape[0], exp_step_factor, T_threshold)
    return fr.render(rays_o.float(), rays_d.float())
