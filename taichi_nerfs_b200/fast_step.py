"""The training step as ONE CUDA graph (no autograd, no host synchronisation, no per-step allocation).

Same math as NGPTrainer.step / the reference's loop body (train.py:184-201) — every stage is one of
the C-ABI kernels, enqueued in a fixed order on fixed buffers:

  [ray-batch sampler] -> ray_aabb -> single-pass march (capacity buffers, one atomic row reservation per ray) ->
  hash fwd (+AABB normalisation) -> fused MLP fwd -> fused per-ray head (composite fwd + background + MSE +
  composite bwd) -> MLP bwd -> hash bwd -> [all-reduce] -> check_finite -> device-side LR/bias-correction update
  -> fused Adam (+fp16 shadow, grad zero) -> device-side GradScaler update

What makes it graph-capturable: the number of samples S stays on the device (kernels read it from the
march counter; buffers are sized for `capacity` rows and rays that would overflow are dropped and
counted), and the per-step optimizer scalars live in device memory.  The reference synchronises the
host on S every step (modules/ray_march.py:187-192) and inside GradScaler.step.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, parallel
from ._lib import F16, F32, check, load
from .fused_mlp import mlp_weights


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class StaticTrainStep:
    def __init__(self, trainer, n_rays: int, samples_per_ray_capacity: int = 384, exp_step_factor: float = 0.0,
                 T_threshold: float = 1e-4, max_samples: int = 1024, use_graph: bool = True,
                 dynamic_loss_scale: bool = True, overlap_optimizer: bool = False, overlap_allreduce=None):
        self.tr = trainer
        m = self.model = trainer.model
        enc = m.pos_encoder
        if not m._fusable(next(m.parameters())):
            raise _lib.NgpError("StaticTrainStep needs the stock NGP architecture (fused MLP)")
        if not hasattr(enc, "hash_table"):
            raise _lib.NgpError("StaticTrainStep runs the hash encoder's kernels; the graph-captured step does not "
                                "support the tri-plane encoder (train it without --graph_step)")
        dev = next(m.parameters()).device
        self.dev, self.n = dev, int(n_rays)
        self.cap = C_ = int(n_rays) * int(samples_per_ray_capacity)
        self.esf, self.T_thr, self.max_samples = float(exp_step_factor), float(T_threshold), int(max_samples)
        self.half = hasattr(enc, "table_f16")
        edt = torch.float16 if self.half else torch.float32
        f32, i32 = torch.float32, torch.int32
        z = lambda *s, dtype=f32: torch.zeros(*s, device=dev, dtype=dtype)  # noqa: E731
        # static inputs
        self.rays_o, self.rays_d, self.gt, self.noise = z(self.n, 3), z(self.n, 3), z(self.n, 3), z(self.n)
        # marching
        self.hits, self.counter, self.rays_a = z(self.n, 2), z(2, dtype=i32), z(self.n, 3, dtype=i32)
        self.xyzs, self.dirs, self.deltas, self.ts = z(C_, 3), z(C_, 3), z(C_), z(C_)
        # network
        self.emb, self.demb = z(C_, 32, dtype=edt), z(C_, 32, dtype=edt)
        self.sig, self.dsig = z(C_), z(C_)
        self.rgbs, self.drgbs = z(C_, 3, dtype=torch.float16), z(C_, 3, dtype=torch.float16)
        self.mlp_save = z(int(load().ngp_mlp_save_bytes(C_)), dtype=torch.uint8)   # h + fp16 rgb kept for the backward
        # compositing / loss
        self.total, self.opacity, self.depth, self.rgb = z(self.n, dtype=i32), z(self.n), z(self.n), z(self.n, 3)
        self.ws = z(C_)
        self.g_rgb, self.g_op, self.g_depth = z(self.n, 3), z(self.n), z(self.n)
        self.loss_sum = z(1)
        # optimizer scalars on the device: owned by the trainer, shared with the module path (NGPTrainer.step)
        self.step_dev, self.hyper, self.scale_state = trainer.step_dev, trainer.hyper, trainer.scale_state
        self.sample_step = torch.full((1,), trainer.step_count, device=dev, dtype=i32)   # batches drawn so far
        # GradScaler state on the device: [scale, growth_tracker (int bits)]; growth 2x / 2000 clean steps, backoff 0.5
        trainer.dynamic_loss_scale = self.dynamic_loss_scale = bool(dynamic_loss_scale)
        self.aabb6 = (C.c_float * 6)(*[float(v) for v in m.xyz_min.flatten().tolist()],
                                     *[float(v) for v in (m.xyz_max - m.xyz_min).flatten().tolist()])
        self._clayout = enc._clayout
        self._w_keep = [w.detach() for w in mlp_weights(m)]
        self._wst = _lib.MlpWeights(*[w.data_ptr() for w in self._w_keep])
        self.P = enc.total_param_size
        assert trainer.slices[0] == (0, self.P), "hash table must be the first parameter"
        offs = [o for o, _ in trainer.slices[1:]]
        assert offs == [self.P, self.P + 2048, self.P + 3072, self.P + 5120, self.P + 9216], offs
        # valid placeholder rays (an all-zero direction would march forever, in the reference too)
        self.rays_o[:] = torch.tensor([1.2, 0.3, 0.5], device=dev)
        jitter = (torch.arange(self.n, device=dev, dtype=f32)[:, None] % 97) * 1e-3
        self.rays_d[:] = -self.rays_o + jitter * torch.tensor([0.3, -0.2, 0.1], device=dev)
        # graphs by (sampled, mode): mode "sync" = forward/backward + optimizer; with overlap_optimizer the optimizer
        # of step k runs at the head of step k+1's graph on a parallel branch next to ray_aabb + marching (which only
        # read the occupancy bitfield): "first" = forward/backward only, "steady" = optimizer(k-1) || march(k), then
        # the network part of step k.  flush() applies the pending update.
        self._graphs, self._kernels = {}, {}
        self.src = None
        self.replays = 0
        self.replays_sampled = 0
        self.graph_kernel_launches = 0   # libngp_b200 kernel nodes executed by graph replays so far
        self.overlap = bool(overlap_optimizer)
        self.pending = False             # gradients of the last step not applied yet (overlap mode only)
        self._side = torch.cuda.Stream(device=dev, priority=-1)
        self._ar_stream = torch.cuda.Stream(device=dev)
        # several ranks, opt-in: all-reduce gradient slices behind the backward kernels that complete them (F = 2 layout)
        import os
        # (opt-in, NGP_AR_OVERLAP=1: on 2 GPUs the three grouped scatter launches + concurrent NCCL kernels cost more
        # than the all-reduce they hide)
        default_ar = ((trainer.world_size > 1 or os.environ.get("NGP_AR_FORCE") == "1") and enc._clayout.feat_dim == 2
                      and os.environ.get("NGP_AR_OVERLAP", "0") == "1")
        self.overlap_allreduce = bool(overlap_allreduce if overlap_allreduce is not None else default_ar)
        if self.overlap_allreduce and getattr(trainer, "p2p", None) is not None:
            self.overlap_allreduce = False   # the peer-memory optimizer step needs no all-reduce at all
        if self.overlap_allreduce and trainer.sharded:
            trainer.sharded = False     # the slice all-reduces replace the reduce-scatter; Adam stays replicated
        # one rank + dynamic loss scale: the backward kernels raise GradScaler's inf flag themselves (a non-finite
        # contribution is seen where it is scattered), the optimizer consumes and clears it - no 45 MB check pass
        self.inf_at_source = bool((trainer.world_size == 1 or trainer.sharded) and self.dynamic_loss_scale
                                  and enc._clayout.feat_dim == 2)
        if self.inf_at_source:
            trainer.found_inf.zero_()
        self.use_graph = bool(use_graph)
        if self.use_graph:
            try:
                # with world_size > 1 the NCCL all-reduce is captured as a graph node too
                for mode in self._modes():
                    self._capture(False, mode)
            except RuntimeError as e:  # pragma: no cover - depends on the NCCL / driver combination
                if parallel.world_info(trainer.pg)[1] == 1:
                    raise
                print(f"[StaticTrainStep] CUDA-graph capture with NCCL failed ({e}); falling back to eager enqueue")
                self._graphs, self._kernels = {}, {}
                self.use_graph = False
                torch.cuda.synchronize()

    def _modes(self):
        return ("first", "steady") if self.overlap else ("sync",)

    # sync-mode views kept for callers that count launches
    @property
    def graph(self):
        return self._graphs.get((False, self._modes()[-1]))

    @property
    def graph_sampled(self):
        return self._graphs.get((True, self._modes()[-1]))

    @property
    def kernels_per_replay(self):
        return self._kernels.get((False, self._modes()[-1]), 0)

    @property
    def kernels_per_replay_sampled(self):
        return self._kernels.get((True, self._modes()[-1]), 0)

    # ---------------------------------------------------------------------------------------------
    def _st(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _table(self):
        return self.tr._shadow if self.half else self.model.pos_encoder.hash_table.data

    def _enqueue_march(self):
        L, m, st, n, cap = load(), self.model, self._st(), self.n, self.cap
        bits = m.density_bitfield
        check(L.ngp_ray_aabb_intersect(_p(self.rays_o), _p(self.rays_d), float(m.scale), _p(self.hits), n, st))
        # single-pass march: every ray reserves its rows with one atomic (row order across rays is arbitrary, as
        # in the reference's atomics at ray_march.py:76-81; the module API keeps the deterministic two-pass layout)
        check(L.ngp_raymarching_frame(_p(self.rays_o), _p(self.rays_d), _p(self.hits), _p(self.noise), _p(bits),
                                      m.cascades, m.grid_size, float(m.scale), self.esf, self.max_samples,
                                      _p(self.counter), _p(self.rays_a), _p(self.xyzs), _p(self.dirs),
                                      _p(self.deltas), _p(self.ts), n, cap, st))

    # the five network kernels, one method each (bench.py times them one by one on the buffers of a real step)
    def _k_hash_fwd(self):
        L, st, tag = load(), self._st(), (F16 if self.half else F32)
        check(L.ngp_hash_encode_fwd_dyn(_p(self.xyzs), _p(self._table()), C.byref(self._clayout), _p(self.emb), tag,
                                        self.cap, _p(self.counter), self.aabb6, st))

    def _k_mlp_fwd(self):
        L, st, tag = load(), self._st(), (F16 if self.half else F32)
        check(L.ngp_mlp_fwd_dyn(_p(self.emb), tag, _p(self.dirs), C.byref(self._wst), _p(self.sig), _p(self.rgbs),
                                _p(self.mlp_save), self.cap, _p(self.counter), st))

    def _k_head(self):
        # composite forward + background + MSE + composite backward in one launch (per-ray work)
        bg = 1.0 if self.esf == 0 else 0.0
        check(load().ngp_ray_head_fused(_p(self.sig), _p(self.rgbs), F16, _p(self.deltas), _p(self.rays_a), _p(self.gt),
                                        bg, float(self.tr.loss_scale),
                                        _p(self.scale_state) if self.dynamic_loss_scale else None, self.T_thr,
                                        _p(self.loss_sum), _p(self.opacity), _p(self.rgb), _p(self.dsig),
                                        _p(self.drgbs), self.n, self._st()))

    def _k_mlp_bwd(self):
        L, st, tag = load(), self._st(), (F16 if self.half else F32)
        gw = self.tr.flat_grad[self.P:self.P + 9408]
        check(L.ngp_mlp_bwd_dyn(_p(self.emb), tag, _p(self.dirs), C.byref(self._wst), _p(self.mlp_save), _p(self.dsig),
                                _p(self.drgbs), _p(self.demb), _p(gw), self.cap, _p(self.counter),
                                _p(self.tr.found_inf) if self.inf_at_source else None, st))

    def _k_hash_bwd(self, level_begin=0, level_end=None):
        L, st, tag = load(), self._st(), (F16 if self.half else F32)
        level_end = self._clayout.n_levels if level_end is None else level_end
        check(L.ngp_hash_encode_bwd_levels(_p(self.xyzs), _p(self.demb), tag, C.byref(self._clayout),
                                           _p(self.tr.flat_grad), self.cap, _p(self.counter), self.aabb6,
                                           int(level_begin), int(level_end),
                                           _p(self.tr.found_inf) if self.inf_at_source else None, st))

    def _level_groups(self):
        """Level groups of the multi-GPU backward, most expensive first: the hashed fine levels (all-distinct cells,
        most atomics), the hashed coarse levels, the dense levels.  Each group owns a contiguous slice of the flat
        gradient buffer (levels are laid out in order)."""
        lay = self._clayout
        L_, first_hashed = lay.n_levels, lay.begin_fast_hash_level
        mid = first_hashed + (L_ - first_hashed) // 2
        groups = [(mid, L_), (first_hashed, mid), (0, first_hashed)]
        return [(a, b) for a, b in groups if b > a]

    def _slice_of_levels(self, a, b):
        lay, F = self._clayout, self._clayout.feat_dim
        lo = lay.offsets[a] * F
        hi = (lay.offsets[b] if b < lay.n_levels else self.P // F) * F
        return lo, hi

    def _enqueue_backward_overlapped(self):
        """Multi-GPU backward: gradient slices are all-reduced on a side stream as soon as they are complete — the MLP
        gradients while the hash scatter runs, each level group while the next group runs — so only the last (small,
        dense-level) slice's all-reduce is exposed (SURVEY.md §8e)."""
        import torch.distributed as dist
        tr, main, ar = self.tr, torch.cuda.current_stream(), self._ar_stream
        fg = tr.flat_grad
        reduce = tr.world_size > 1     # (a single rank can still run the grouped launches: tests)

        def allreduce_behind(lo, hi):
            ar.wait_stream(main)
            with torch.cuda.stream(ar):
                dist.all_reduce(fg[lo:hi], group=tr.pg)
        self._k_mlp_bwd()
        if reduce:
            allreduce_behind(self.P, fg.numel())                        # MLP weight gradients (37.6 KB)
        for a, b in self._level_groups():
            self._k_hash_bwd(a, b)
            if reduce:
                allreduce_behind(*self._slice_of_levels(a, b))
        if reduce:
            main.wait_stream(ar)

    def _enqueue_network(self):
        # counter[0] = number of valid sample rows, read on the device by every kernel
        self._k_hash_fwd()
        self._k_mlp_fwd()
        self._k_head()
        if self.overlap_allreduce:
            self._enqueue_backward_overlapped()
        else:
            self._k_mlp_bwd()
            self._k_hash_bwd()

    def _enqueue_sampler(self):
        """datasets/base.py:34-61 + ray_utils.py:51-80 + the marching jitter, keyed by (seed, batch counter, ray)."""
        src = self.src
        check(load().ngp_sample_ray_batch(_p(src["bank"]), src["bank"].shape[2], _p(src["poses"]), _p(src["dirs"]),
                                          src["poses"].shape[0], src["dirs"].shape[0], None, None, src["fixed_img"],
                                          src["seed"], _p(self.sample_step), 0, _p(self.rays_o), _p(self.rays_d),
                                          _p(self.gt), _p(self.noise), None, None, self.n, self._st()))

    def _enqueue_update(self):
        # [all-reduce, unless the backward already reduced slice by slice] -> check_finite -> LR/bias scalars ->
        # fused Adam -> GradScaler.update
        self.tr.enqueue_update(allreduce=not self.overlap_allreduce, check_finite=not self.inf_at_source)

    def _enqueue(self, sampled=False, mode="sync"):
        if sampled:
            self._enqueue_sampler()
        # march counter, loss accumulator, found_inf <- 0 and (own batch counter: step_dev moves with the optimizer,
        # which may run a step late) sample_step += 1, in one launch
        # (with inf_at_source the flag is raised by the previous backward and cleared by its consumer, the optimizer)
        check(load().ngp_step_reset(_p(self.counter), _p(self.loss_sum),
                                    None if self.inf_at_source else _p(self.tr.found_inf),
                                    _p(self.sample_step) if sampled else None, self._st()))
        if mode == "steady":
            # optimizer of the PREVIOUS step beside this step's ray_aabb + marching.  The marching branch runs on
            # a high-priority stream (the priority is kept by the captured kernel nodes): its latency-bound warps
            # take SM slots first and the bandwidth-bound Adam sweep fills in around them.
            main = torch.cuda.current_stream()
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                self._enqueue_march()
            self._enqueue_update()
            main.wait_stream(self._side)
            self._enqueue_network()
            return
        self._enqueue_march()
        self._enqueue_network()
        if mode == "sync":
            self._enqueue_update()

    def _capture(self, sampled, mode):
        # the graph must not mutate training state while being built: snapshot, warm up + capture, restore
        tr = self.tr
        keep = [p.data.clone() for p in tr.params] + [tr.exp_avg.clone(), tr.exp_avg_sq.clone(), self.step_dev.clone()]
        scale_keep, hyper_keep, sample_keep = self.scale_state.clone(), self.hyper.clone(), self.sample_step.clone()
        shadow = None if tr._shadow_full is None else tr._shadow_full.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._enqueue(sampled, mode)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        before = _lib.launch_count()
        with torch.cuda.graph(graph):
            self._enqueue(sampled, mode)
        kernels = _lib.launch_count() - before  # libngp_b200 kernel nodes in the graph
        torch.cuda.synchronize()
        for p, k in zip(tr.params, keep):
            p.data.copy_(k)
        tr.exp_avg.copy_(keep[-3])
        tr.exp_avg_sq.copy_(keep[-2])
        self.step_dev.copy_(keep[-1])
        self.scale_state.copy_(scale_keep)
        self.hyper.copy_(hyper_keep)
        self.sample_step.copy_(sample_keep)
        tr.flat_grad.zero_()
        if shadow is not None:
            tr._shadow_full.copy_(shadow)
        self._graphs[(sampled, mode)], self._kernels[(sampled, mode)] = graph, kernels

    # ---------------------------------------------------------------------------------------------
    def step(self, rays_o, rays_d, rgb_gt, noise=None):
        """Enqueues one full training step; returns the (device) loss tensor — nothing is synchronised."""
        self.rays_o.copy_(rays_o, non_blocking=True)
        self.rays_d.copy_(rays_d, non_blocking=True)
        self.gt.copy_(rgb_gt, non_blocking=True)
        if noise is None:
            self.noise.uniform_()
        else:
            self.noise.copy_(noise, non_blocking=True)
        self._run(False)
        self.replays += 1 if self.use_graph else 0
        return self._finish_step()

    def _run(self, sampled):
        mode = "sync" if not self.overlap else ("steady" if self.pending else "first")
        if self.use_graph:
            self._graphs[(sampled, mode)].replay()
            self.graph_kernel_launches += self._kernels[(sampled, mode)]
        else:
            self._enqueue(sampled, mode)
        self.pending = self.overlap
        if getattr(self.tr, 'sharded', False):
            self.tr.master_stale = True     # (the Python side of the update does not run on a graph replay)

    def flush(self):
        """Overlap mode: apply the optimizer update of the last step now (before anything reads the parameters:
        update_density_grid, rendering, checkpoints).  No-op otherwise."""
        if self.pending:
            if not self.inf_at_source:
                self.tr.found_inf.zero_()
            self._enqueue_update()
            self.pending = False
            if self.tr._shadow is not None:
                self.model.pos_encoder.adopt_shadow(self.tr._shadow)
        self.tr.sync_master()   # sharded optimizer: the fp32 master table is complete again on every rank

    def _finish_step(self):
        self.tr.step_count += 1
        enc = self.model.pos_encoder
        if self.tr._shadow is not None:
            enc.adopt_shadow(self.tr._shadow)
        return self.loss_sum / (3.0 * self.n)

    def attach_ray_source(self, image_bank, poses, directions, seed: int = 0, fixed_img: int = -1):
        """Keep the training set resident (as the reference's ``train_dataset.to(device)``) and let the step draw
        its own batch: ``step_sampled()`` then needs no per-step input at all.  With several ranks pass a
        different ``seed`` per rank."""
        f = lambda t: t.detach().to(self.dev, torch.float32).contiguous()  # noqa: E731
        bank, poses, directions = f(image_bank), f(poses), f(directions)
        if bank.ndim != 3 or bank.shape[0] != poses.shape[0] or bank.shape[1] != directions.shape[0] or bank.shape[2] < 3:
            raise ValueError(f"image bank {tuple(bank.shape)} vs {poses.shape[0]} poses x {directions.shape[0]} pixels")
        self.src = dict(bank=bank, poses=poses.reshape(-1, 3, 4), dirs=directions, seed=int(seed),
                        fixed_img=int(fixed_img))
        if self.use_graph:
            self.flush()
            for mode in self._modes():
                self._capture(True, mode)
        return self

    def step_sampled(self):
        """One training step on a batch drawn on the device (no host input, no host sync)."""
        if self.src is None:
            raise _lib.NgpError("step_sampled() needs attach_ray_source() first")
        self._run(True)
        self.replays_sampled += 1 if self.use_graph else 0
        return self._finish_step()

    def stats(self):
        """(samples marched, rays) of the LAST enqueued step — device tensors, no sync."""
        return self.counter[0], self.counter[1]
