"""The training step as ONE CUDA graph (no autograd, no host synchronisation, no per-step allocation).

Same math as NGPTrainer.step / the reference's loop body (train.py:184-201) — every stage is one of
the C-ABI kernels, enqueued in a fixed order on fixed buffers:

  [ray-batch sampler] -> ray_aabb -> single-pass march (capacity buffers, one atomic row reservation per ray) ->
  hash (or tri-plane) fwd (+AABB normalisation) -> fused MLP fwd -> fused per-ray head (composite fwd + background + MSE
  [+ distortion loss] [+ depth loss] + composite bwd) -> MLP bwd -> hash (or tri-plane) bwd -> [gradient exchange] -> check_finite -> device-side LR/bias-correction update
  -> fused Adam (+fp16 shadow, grad zero) -> device-side GradScaler update

With camera extrinsics refinement (DESIGN.md §6i) the rays come from the pose-apply kernel (the graph's first node, on
camera directions and image indices), the hash backward is followed by the position gradient and the pose gradient,
and the corrections' Adam runs next to the model's.

With camera intrinsics refinement (DESIGN.md §6l) the step's first nodes after the reset are the camera unproject (the
rays' camera directions from their pixels under the corrected intrinsics, which also clears the per-ray gradient rows)
and the pose apply (with the extrinsics corrections, or a zero buffer); the hash backward is followed by the one
position-gradient pass and the intrinsics gradient, and the intrinsics Adam runs next to the model's.

With error-map sampling (DESIGN.md §6j) each ray carries a weight w_r: the head is followed by the error-map accumulate
(the rays' errors into their tiles) and by the gradient weight (every per-sample gradient of ray r times w_r), so the
backward sees the gradient of the weighted loss; loss_sum, the logged value, stays the unweighted one.  The sampled step
draws its pixels with the error-map sampler, whose indices the batch sampler then reads.

With exposure compensation (DESIGN.md §6k) the exposure apply runs between the network (or voxel) forward and the head,
which reads its scaled copy of the sample colours; the exposure backward runs after the head (and the error-map nodes),
rewriting the per-sample colour gradient before the network backward, and the exposures' Adam runs next to the model's.

A voxel-grid model (--model_name svox) has no network: the march feeds the voxel forward (fp32 sigma / rgb) -> head ->
voxel backward -> [regularisers] -> finite check and Adam over the fields' node block B only (DESIGN.md §6b).

What makes it graph-capturable: the number of samples S stays on the device (kernels read it from the
march counter; buffers are sized for `capacity` rows and rays that would overflow are dropped and
counted), and the per-step optimizer scalars live in device memory.  The reference synchronises the
host on S every step (modules/ray_march.py:187-192) and inside GradScaler.step.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, ops, parallel
from ._lib import F16, F32, check, load
from .fused_mlp import mlp_weights


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class StaticTrainStep:
    def __init__(self, trainer, n_rays: int, samples_per_ray_capacity: int = 384, exp_step_factor: float = 0.0,
                 T_threshold: float = 1e-4, max_samples: int = 1024, use_graph: bool = True,
                 dynamic_loss_scale: bool = True, overlap_optimizer: bool = False, distortion_loss_w: float = 0.0,
                 random_bg: bool = False, bg_seed: int = 0, bg_load: float = 1.0, depth_loss_w: float = 0.0,
                 extrinsics=None, error_map=None):
        self.tr = trainer
        m = self.model = trainer.model
        # the voxel-grid model: fp32 fields and outputs, no encoder and no MLP; its optimizer pass covers the node
        # block B only (DESIGN.md §6b).  Otherwise the two encoder stages are the encoder's launches (hash or
        # tri-plane), with its embedding dtype.
        enc = self.enc = trainer.encoder
        self.vox = enc is None
        if self.vox:
            if trainer.world_size > 1:
                raise _lib.NgpError("StaticTrainStep runs a voxel-grid model on one rank only")
        elif not m._fusable(next(m.parameters())):
            raise _lib.NgpError("StaticTrainStep needs the stock NGP architecture (fused MLP)")
        # extrinsics: the trainer's PoseRefinement (NGPTrainer(extrinsics=...)), shared with the module path, or None
        if extrinsics is not trainer.extrinsics:
            raise ValueError("StaticTrainStep: extrinsics must be the trainer's PoseRefinement "
                             "(NGPTrainer(extrinsics=...)), or None for a trainer without one")
        self.ext = extrinsics
        # intrinsics: the trainer's IntrinsicsRefinement (NGPTrainer(intrinsics=...)), shared with the module path
        self.intr = trainer.intrinsics
        if self.intr is not None:
            if overlap_optimizer:
                raise _lib.NgpError("StaticTrainStep: intrinsics refinement does not combine with overlap_optimizer "
                                    "(the next step's march would read intrinsics one update stale)")
            if trainer.world_size > 1:
                raise _lib.NgpError("StaticTrainStep: intrinsics refinement runs on one rank")
        # error_map: a taichi_nerfs_b200.error_map.ErrorMap over the training images, or None (nothing is enqueued)
        self.em = error_map
        # exposure compensation: the trainer's ExposureCorrection (NGPTrainer(exposure=...)), shared with the module path
        self.expo = trainer.exposure
        if self.ext is not None and overlap_optimizer:
            raise _lib.NgpError("StaticTrainStep: extrinsics refinement does not combine with overlap_optimizer (the "
                                "next step's march would read poses one update stale)")
        dev = next(m.parameters()).device
        self.dev, self.n = dev, int(n_rays)
        self.cap = C_ = int(n_rays) * int(samples_per_ray_capacity)
        self.esf, self.T_thr, self.max_samples = float(exp_step_factor), float(T_threshold), int(max_samples)
        # weight of the distortion loss (train.py --distortion_loss_w): loss = mse + w * mean(distortion per ray)
        self.distortion_w = float(distortion_loss_w)
        if not self.distortion_w >= 0.0 or self.distortion_w == float("inf"):
            raise ValueError(f"distortion_loss_w must be finite and >= 0, got {distortion_loss_w}")
        # weight of the depth loss (train.py --depth_loss_w, DESIGN.md §6h): loss += w * mean(v (D - D^)^2)
        self.depth_w = float(depth_loss_w)
        if not self.depth_w >= 0.0 or self.depth_w == float("inf"):
            raise ValueError(f"depth_loss_w must be finite and >= 0, got {depth_loss_w}")
        # fp16 embeddings (the --half_opt hash encoder): the MLP kernels run their fp16-embedding instantiations
        self.half = not self.vox and enc.emb_dtype == torch.float16
        edt = torch.float16 if self.half else torch.float32
        f32, i32 = torch.float32, torch.int32
        z = lambda *s, dtype=f32: torch.zeros(*s, device=dev, dtype=dtype)  # noqa: E731
        # static inputs
        self.rays_o, self.rays_d, self.gt, self.noise = z(self.n, 3), z(self.n, 3), z(self.n, 3), z(self.n)
        # marching
        self.hits, self.counter, self.rays_a = z(self.n, 2), z(2, dtype=i32), z(self.n, 3, dtype=i32)
        self.xyzs, self.dirs, self.deltas, self.ts = z(C_, 3), z(C_, 3), z(C_), z(C_)
        # network (the voxel grid: sigma and fp32 rgb straight from the fields, no embedding)
        self.sig, self.dsig = z(C_), z(C_)
        if self.vox:
            self.emb = self.demb = self.mlp_save = None
            self.rgbs, self.drgbs = z(C_, 3), z(C_, 3)
        else:
            self.emb, self.demb = z(C_, 32, dtype=edt), z(C_, 32, dtype=edt)
            self.rgbs, self.drgbs = z(C_, 3, dtype=torch.float16), z(C_, 3, dtype=torch.float16)
            self.mlp_save = z(int(load().ngp_mlp_save_bytes(C_)), dtype=torch.uint8)   # h + fp16 rgb for the backward
        # compositing / loss
        self.total, self.opacity, self.depth, self.rgb = z(self.n, dtype=i32), z(self.n), z(self.n), z(self.n, 3)
        self.ws = z(C_)
        self.g_rgb, self.g_op, self.g_depth = z(self.n, 3), z(self.n), z(self.n)
        self.loss_sum = z(1)
        # optimizer scalars on the device: owned by the trainer, shared with the module path (NGPTrainer.step)
        self.step_dev, self.hyper, self.scale_state = trainer.step_dev, trainer.hyper, trainer.scale_state
        self.sample_step = torch.full((1,), trainer.step_count, device=dev, dtype=i32)   # batches drawn so far
        # --random_bg (DESIGN.md §6f): per-ray background colours of step s drawn on the device; s = bg_step[0], which
        # the step's reset launch increments, so s = trainer.step_count after the step (as ops.random_bg is called by
        # the module path).  alpha stays 1 (target unchanged) when step() gets no alpha.
        self.random_bg, self.bg_seed, self.bg_load = bool(random_bg), int(bg_seed), float(bg_load)
        self.bg_step = torch.full((1,), trainer.step_count, device=dev, dtype=i32)
        self.bg_rgb, self.alpha = (z(self.n, 3), torch.ones(self.n, device=dev)) if self.random_bg else (None, None)
        self.depth_gt = z(self.n) if self.depth_w > 0 else None   # per-ray target z-depth, 0 = none
        # extrinsics refinement: camera directions and image indices in, dL/dx of every sample row
        if self.ext is not None or self.intr is not None:
            self.cam_dirs, self.img_idx = z(self.n, 3), torch.zeros(self.n, device=dev, dtype=torch.int64)
            self.cam_dirs[:, 2] = -1.0   # valid placeholder rays for the capture (a zero direction never advances)
            self.dx = z(C_, 3)
        if self.intr is not None:
            # each ray's pixel; the pose apply's corrections when extrinsics refinement is off (zero: the rays of
            # get_rays bit for bit, DESIGN.md §6i)
            self.pix = torch.zeros(self.n, device=dev, dtype=torch.int64)
            self.pose_corr = self.ext.corr if self.ext is not None else z(self.intr.n_img, 8)
            self.intr.reserve(self.n)
            self.intr.n_rays = self.n
        if self.em is not None:   # each ray's image, pixel and loss weight
            self.em_img = torch.zeros(self.n, device=dev, dtype=torch.int64)
            self.em_pix = self.pix if self.intr is not None else torch.zeros(self.n, device=dev, dtype=torch.int64)
            self.ray_w = torch.ones(self.n, device=dev)
        if self.expo is not None:
            # the head's copy of the sample colours under their images' gains; each ray's image is the index buffer
            # extrinsics refinement or the error map fill, else one of its own (step(img_idxs=...) or the sampler)
            self.rgbs_expo = torch.zeros_like(self.rgbs)
            self.expo_img = (self.img_idx if self.ext is not None or self.intr is not None
                             else self.em_img if self.em is not None
                             else torch.zeros(self.n, device=dev, dtype=torch.int64))
        self._head_rgbs = self.rgbs_expo if self.expo is not None else self.rgbs
        # GradScaler state on the device: [scale, growth_tracker (int bits)]; growth 2x / 2000 clean steps, backoff 0.5
        trainer.dynamic_loss_scale = self.dynamic_loss_scale = bool(dynamic_loss_scale)
        self.aabb6 = (C.c_float * 6)(*[float(v) for v in m.xyz_min.flatten().tolist()],
                                     *[float(v) for v in (m.xyz_max - m.xyz_min).flatten().tolist()])
        if self.vox:
            # B: the nodes the step's samples (inside the scene box, with one node of margin) and the regularisers
            # reach.  The step's optimizer checks and updates B only; see DESIGN.md §6b for mixed use with the module
            # path.
            self._clayout = m._clayout
            self.block = tuple(int(v) for v in m._reg_block)
            self.P = m.sh_fields.numel()
            assert trainer.slices[0] == (0, self.P) and trainer.slices[1][1] == m.density_fields.numel()
        else:
            self._w_keep = [w.detach() for w in mlp_weights(m)]
            self._wst = _lib.MlpWeights(*[w.data_ptr() for w in self._w_keep])
            self.P = enc.total_param_size
            assert trainer.slices[0] == (0, self.P), "the encoder's table must be the first parameter"
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
        # one rank or the peer-memory step + dynamic loss scale: the backward kernels raise GradScaler's inf flag
        # themselves (a non-finite contribution is seen where it is scattered), the optimizer consumes and clears it -
        # no 45 MB check pass (the NCCL fallback checks the reduced fp16 sum instead)
        # (enc.bwd_raises_inf: the hash backward raises it in its F = 2 instantiation only, the tri-plane backward in
        # both).  The voxel grid: the regularisers' gradient is not seen by any backward, so the finite check over B
        # covers them all.
        self.inf_at_source = bool((trainer.world_size == 1 or trainer.p2p is not None) and self.dynamic_loss_scale
                                  and not self.vox and enc.bwd_raises_inf)
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
        # the fp16 hash table: the trainer's shadow slice, which the fused Adam rewrites in place (the encoder's own
        # kernel_table() re-casts into a new tensor whenever the master moved); else a view of the trainer's flat_param
        return self.tr._shadow if self.tr._shadow is not None else self.enc.kernel_table()

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
    # (the two _k_hash_* are "the position encoder": hash or tri-plane, they run the encoder's launches)
    def _k_hash_fwd(self):
        check(self.enc.enqueue_encode_dyn(load(), _p(self.xyzs), _p(self._table()), _p(self.emb), self.cap,
                                          _p(self.counter), self.aabb6, self._st()))

    def _k_mlp_fwd(self):
        L, st, tag = load(), self._st(), (F16 if self.half else F32)
        check(L.ngp_mlp_fwd_dyn(_p(self.emb), tag, _p(self.dirs), C.byref(self._wst), _p(self.sig), _p(self.rgbs),
                                _p(self.mlp_save), self.cap, _p(self.counter), st))

    def _k_head(self):
        # composite forward + background + MSE [+ distortion loss] [+ depth loss] + composite backward in one launch
        # (per-ray work)
        bg = 1.0 if self.esf == 0 else 0.0
        ctag = F32 if self.vox else F16
        if self.random_bg:
            L, st = load(), self._st()
            check(L.ngp_random_bg(self.bg_seed & 0xFFFFFFFFFFFFFFFF, _p(self.bg_step), 0, _p(self.bg_rgb), self.n, st))
        if self.depth_w > 0:
            check(load().ngp_ray_head_fused_depth(
                _p(self.sig), _p(self._head_rgbs), ctag, _p(self.deltas), _p(self.ts), _p(self.rays_a), _p(self.gt),
                bg, _p(self.bg_rgb), _p(self.alpha), self.bg_load, float(self.tr.loss_scale),
                _p(self.scale_state) if self.dynamic_loss_scale else None, self.T_thr, self.distortion_w,
                _p(self.depth_gt), self.depth_w, _p(self.loss_sum), _p(self.opacity), _p(self.rgb), _p(self.dsig),
                _p(self.drgbs), self.n, self._st()))
            return
        if self.random_bg:
            check(L.ngp_ray_head_fused_random_bg(
                _p(self.sig), _p(self._head_rgbs), ctag, _p(self.deltas), _p(self.ts), _p(self.rays_a), _p(self.gt),
                _p(self.bg_rgb), _p(self.alpha), self.bg_load, float(self.tr.loss_scale),
                _p(self.scale_state) if self.dynamic_loss_scale else None, self.T_thr, self.distortion_w,
                _p(self.loss_sum), _p(self.opacity), _p(self.rgb), _p(self.dsig), _p(self.drgbs), self.n, st))
            return
        if self.distortion_w > 0:
            check(load().ngp_ray_head_fused_distortion(
                _p(self.sig), _p(self._head_rgbs), ctag, _p(self.deltas), _p(self.ts), _p(self.rays_a), _p(self.gt),
                bg, float(self.tr.loss_scale), _p(self.scale_state) if self.dynamic_loss_scale else None, self.T_thr,
                self.distortion_w, _p(self.loss_sum), _p(self.opacity), _p(self.rgb), _p(self.dsig), _p(self.drgbs),
                self.n, self._st()))
            return
        check(load().ngp_ray_head_fused(_p(self.sig), _p(self._head_rgbs), ctag, _p(self.deltas), _p(self.rays_a),
                                        _p(self.gt), bg, float(self.tr.loss_scale),
                                        _p(self.scale_state) if self.dynamic_loss_scale else None, self.T_thr,
                                        _p(self.loss_sum), _p(self.opacity), _p(self.rgb), _p(self.dsig),
                                        _p(self.drgbs), self.n, self._st()))

    def _k_mlp_bwd(self):
        L, st, tag = load(), self._st(), (F16 if self.half else F32)
        gw = self.tr.flat_grad[self.P:self.P + 9408]
        check(L.ngp_mlp_bwd_dyn(_p(self.emb), tag, _p(self.dirs), C.byref(self._wst), _p(self.mlp_save), _p(self.dsig),
                                _p(self.drgbs), _p(self.demb), _p(gw), self.cap, _p(self.counter),
                                _p(self.tr.found_inf) if self.inf_at_source else None, st))

    def _k_hash_bwd(self):
        check(self.enc.enqueue_encode_bwd_dyn(load(), _p(self.xyzs), _p(self._table()), _p(self.demb),
                                              _p(self.tr.flat_grad), self.cap, _p(self.counter), self.aabb6,
                                              _p(self.tr.found_inf) if self.inf_at_source else None, self._st()))

    # extrinsics refinement (DESIGN.md §6i): rays from the corrected poses; dL/dx of the rows; the pose gradient
    def _k_pose_apply(self):
        e = self.ext
        check(load().ngp_pose_apply(_p(self.cam_dirs), _p(self.img_idx), _p(e.poses), _p(e.corr), e.n_img,
                                    _p(self.rays_o), _p(self.rays_d), self.n, self._st()))

    def _k_hash_dx(self):
        check(load().ngp_hash_encode_bwd_input_dyn(_p(self.xyzs), _p(self._table()), _p(self.demb),
                                                   self.enc._tag(), C.byref(self.enc._clayout), _p(self.dx),
                                                   self.cap, _p(self.counter), self.aabb6, self._st()))

    # intrinsics refinement (DESIGN.md §6l): the rays' camera directions from their pixels; the intrinsics gradient
    def _k_unproject(self):
        i = self.intr
        model, params = ops._camera_args(i.camera)
        check(load().ngp_camera_unproject(_p(self.pix), self.n, i.W, i.H, model, params, _p(i.corr), _p(self.cam_dirs),
                                          _p(i.grad_rays), None, _p(self.tr.found_inf), self._st()))

    def _k_pose_apply_intr(self):
        i = self.intr
        check(load().ngp_pose_apply(_p(self.cam_dirs), _p(self.img_idx), _p(i.poses), _p(self.pose_corr), i.n_img,
                                    _p(self.rays_o), _p(self.rays_d), self.n, self._st()))

    def _k_intr_grad(self):
        i = self.intr
        model, params = ops._camera_args(i.camera)
        check(load().ngp_intrinsics_grad(_p(self.dx), _p(self.ts), _p(self.rays_a), self.n, None, self.cap,
                                         _p(self.pix), _p(self.img_idx), _p(i.poses),
                                         _p(self.ext.corr) if self.ext is not None else None, i.n_img,
                                         _p(self.cam_dirs), i.W, i.H, model, params, _p(i.corr), _p(i.grad_rays),
                                         self.n, _p(self.tr.found_inf), self._st()))

    def _k_pose_grad(self):
        e = self.ext
        check(load().ngp_pose_grad(_p(self.dx), _p(self.ts), _p(self.rays_a), _p(self.img_idx), _p(self.rays_d),
                                   self.n, None, self.cap, e.n_img, _p(e.grad), _p(self.tr.found_inf), self._st()))

    # the voxel grid's stages: fields -> fp32 sigma / rgb, and the field gradient into the trainer's flat buffer
    def _k_voxel_fwd(self):
        m = self.model
        check(load().ngp_voxel_fwd_dyn(_p(self.xyzs), _p(self.dirs), _p(m.sh_fields), _p(m.density_fields),
                                       C.byref(self._clayout), _p(self.sig), _p(self.rgbs), self.cap, _p(self.counter),
                                       self._st()))

    def _k_voxel_bwd(self):
        dsh, dden = self.model.grad_sink
        check(load().ngp_voxel_bwd_dyn(_p(self.xyzs), _p(self.dirs), _p(self.sig), _p(self.rgbs), _p(self.dsig),
                                       _p(self.drgbs), C.byref(self._clayout), _p(dsh), _p(dden), self.cap,
                                       _p(self.counter), None, self._st()))

    # error-map sampling (DESIGN.md §6j): the rays' errors into the map, then the per-ray loss weights
    def _k_em_accumulate(self):
        em = self.em
        rbg = self.random_bg
        check(load().ngp_error_map_accumulate(_p(self.rgb), _p(self.gt), _p(self.bg_rgb) if rbg else None,
                                              _p(self.alpha) if rbg else None, self.bg_load, _p(self.em_img),
                                              _p(self.em_pix), *em.geom, _p(em.acc), _p(em.cnt), self.n, self._st()))

    def _k_grad_weight(self):
        check(load().ngp_ray_grad_weight(_p(self.rays_a), _p(self.ray_w), _p(self.dsig), _p(self.drgbs),
                                         F32 if self.vox else F16, _p(self.tr.found_inf), self.n, self.cap, self._st()))

    # exposure compensation (DESIGN.md §6k): the colours the head reads; the colour gradient and the exposure gradient
    def _k_expo_apply(self):
        x = self.expo
        check(load().ngp_exposure_apply(_p(self.rgbs), F32 if self.vox else F16, _p(self.rays_a), _p(self.expo_img),
                                        _p(x.exposure), x.n_img, _p(self.rgbs_expo), self.n, self.cap,
                                        _p(self.counter), self._st()))

    def _k_expo_bwd(self):
        x = self.expo
        check(load().ngp_exposure_bwd(_p(self.rgbs_expo), _p(self.drgbs), F32 if self.vox else F16, _p(self.rays_a),
                                      _p(self.expo_img), _p(x.exposure), x.n_img, _p(x.grad), _p(self.tr.found_inf),
                                      self.n, self.cap, _p(self.counter), self._st()))

    def _k_head_weighted(self):
        self._k_head()
        if self.em is not None:
            self._k_em_accumulate()
            self._k_grad_weight()

    def _k_head_exposed(self):
        if self.expo is not None:
            self._k_expo_apply()
        self._k_head_weighted()
        if self.expo is not None:
            self._k_expo_bwd()

    def _enqueue_network(self):
        # counter[0] = number of valid sample rows, read on the device by every kernel
        if self.vox:
            self._k_voxel_fwd()
            self._k_head_exposed()
            self._k_voxel_bwd()
            if self.tr.voxel_reg is not None:   # TV / sparsity over B, scaled by the device loss scale
                self.tr.add_voxel_reg()
            return
        self._k_hash_fwd()
        self._k_mlp_fwd()
        self._k_head_exposed()
        self._k_mlp_bwd()
        self._k_hash_bwd()
        if self.ext is not None or self.intr is not None:   # one position-gradient pass feeds both
            self._k_hash_dx()
        if self.ext is not None:
            self._k_pose_grad()
        if self.intr is not None:
            self._k_intr_grad()

    def _enqueue_sampler(self):
        """datasets/base.py:34-61 + ray_utils.py:51-80 + the marching jitter, keyed by (seed, batch counter, ray)."""
        src = self.src
        em, img, pix = self.em, None, None
        if em is not None:   # the pixels come from the error map; the batch sampler gathers them
            check(load().ngp_error_map_sample(_p(em.cdf), *em.geom, em.seed & 0xFFFFFFFFFFFFFFFF, _p(self.sample_step),
                                              0, _p(self.em_img), _p(self.em_pix), _p(self.ray_w), self.n, self._st()))
            img, pix = _p(self.em_img), _p(self.em_pix)
        check(load().ngp_sample_ray_batch(_p(src["bank"]), src["bank"].shape[2], _p(src["poses"]), _p(src["dirs"]),
                                          src["poses"].shape[0], src["dirs"].shape[0], img, pix, src["fixed_img"],
                                          src["seed"], _p(self.sample_step), 0, _p(self.rays_o), _p(self.rays_d),
                                          _p(self.gt), _p(self.noise),
                                          _p(self.expo_img) if self.expo is not None and em is None else None, None,
                                          self.n, self._st()))

    def _enqueue_update(self):
        # [gradient exchange] -> check_finite -> LR/bias scalars -> fused Adam -> GradScaler.update
        self.tr.enqueue_update(check_finite=not self.inf_at_source, voxel_block=self.block if self.vox else None)

    def _enqueue(self, sampled=False, mode="sync"):
        if self.ext is not None and self.intr is None:
            self._k_pose_apply()
        if sampled:
            self._enqueue_sampler()
        # march counter, loss accumulator, found_inf <- 0 and (own batch counter: step_dev moves with the optimizer,
        # which may run a step late) sample_step += 1, in one launch
        # (with inf_at_source the flag is raised by the previous backward and cleared by its consumer, the optimizer)
        check(load().ngp_step_reset(_p(self.counter), _p(self.loss_sum),
                                    None if self.inf_at_source else _p(self.tr.found_inf),
                                    _p(self.sample_step) if sampled else _p(self.bg_step) if self.random_bg else None,
                                    self._st()))
        if self.intr is not None:   # after the reset: a pixel that is not invertible raises found_inf for this step
            self._k_unproject()
            self._k_pose_apply_intr()
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
        bg_step_keep = self.bg_step.clone()
        ext_keep = [] if self.ext is None else [t.clone() for t in self.ext.state()]
        em_keep = [] if self.em is None else [t.clone() for t in self.em.state()]
        expo_keep = [] if self.expo is None else [t.clone() for t in self.expo.state()]
        intr_keep = [] if self.intr is None else [t.clone() for t in self.intr.state()]
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
        self.bg_step.copy_(bg_step_keep)
        if self.ext is not None:
            for t, k in zip(self.ext.state(), ext_keep):
                t.copy_(k)
        if self.em is not None:
            for t, k in zip(self.em.state(), em_keep):
                t.copy_(k)
        if self.expo is not None:
            for t, k in zip(self.expo.state(), expo_keep):
                t.copy_(k)
        if self.intr is not None:
            for t, k in zip(self.intr.state(), intr_keep):
                t.copy_(k)
        tr.flat_grad.zero_()
        if shadow is not None:
            tr._shadow_full.copy_(shadow)
        self._graphs[(sampled, mode)], self._kernels[(sampled, mode)] = graph, kernels

    # ---------------------------------------------------------------------------------------------
    def step(self, rays_o, rays_d, rgb_gt, noise=None, alpha=None, depth=None, directions=None, img_idxs=None,
             ray_w=None, pix_idxs=None):
        """Enqueues one full training step; returns the (device) loss tensor — nothing is synchronised.  ``alpha`` [N]
        (random_bg only): the images' alpha, whose transparent part of the target gets the ray's colour.  ``depth`` [N]
        (depth_loss_w > 0 only, where it is required): each ray's target z-depth, 0 where there is none.  With
        extrinsics refinement the step forms its rays itself: rays_o and rays_d are None and ``directions`` [N, 3]
        (camera frame) and ``img_idxs`` [N] (or one index for the whole batch) are required.  With an error map,
        ``ray_w`` [N] (the loss weights of ErrorMap.draw), ``img_idxs`` and ``pix_idxs`` [N] are required.  With exposure
        compensation ``img_idxs`` [N] (or one index) is required.  With intrinsics refinement the step forms its rays
        from pixels: rays_o, rays_d and ``directions`` are None, and ``img_idxs`` and ``pix_idxs`` [N] are required."""
        if self.expo is not None and img_idxs is None:
            raise ValueError("exposure compensation: step(..., img_idxs=...) (each ray's image, whose gain its samples "
                             "take)")
        if self.intr is not None:
            if pix_idxs is None or img_idxs is None or rays_o is not None or rays_d is not None or \
                    directions is not None:
                raise ValueError("intrinsics refinement: step(None, None, rgb, ..., img_idxs=..., pix_idxs=...) (the "
                                 "step forms the rays from the pixels under the corrected intrinsics)")
            self.pix.copy_(torch.as_tensor(pix_idxs, device=self.dev).reshape(-1), non_blocking=True)
            self.img_idx.copy_(torch.as_tensor(img_idxs, device=self.dev).reshape(-1), non_blocking=True)
        if self.em is not None:
            if ray_w is None or img_idxs is None or pix_idxs is None:
                raise ValueError("error-map sampling: step(..., ray_w=..., img_idxs=..., pix_idxs=...) (the rays' loss "
                                 "weights and the tiles their errors go to)")
            self.ray_w.copy_(ray_w, non_blocking=True)
            self.em_img.copy_(torch.as_tensor(img_idxs, device=self.dev).reshape(-1), non_blocking=True)
            self.em_pix.copy_(pix_idxs, non_blocking=True)
        elif ray_w is not None or (pix_idxs is not None and self.intr is None):
            raise ValueError("ray_w / pix_idxs are read by error-map sampling only (StaticTrainStep(error_map=...))")
        if self.intr is not None:
            pass
        elif self.ext is not None:
            if directions is None or img_idxs is None or rays_o is not None or rays_d is not None:
                raise ValueError("extrinsics refinement: step(None, None, rgb, ..., directions=..., img_idxs=...) "
                                 "(the step forms the rays from the corrected poses)")
            self.cam_dirs.copy_(directions, non_blocking=True)
            self.img_idx.copy_(torch.as_tensor(img_idxs, device=self.dev).reshape(-1), non_blocking=True)
        elif directions is not None or (img_idxs is not None and self.em is None and self.expo is None):
            raise ValueError("directions / img_idxs are read by extrinsics refinement, error-map sampling and exposure "
                             "compensation only (StaticTrainStep(extrinsics=... | error_map=...), "
                             "NGPTrainer(exposure=...))")
        elif self.expo is not None and self.em is None:   # the step's own index buffer
            self.expo_img.copy_(torch.as_tensor(img_idxs, device=self.dev).reshape(-1), non_blocking=True)
        if depth is None and self.depth_w > 0:
            raise ValueError("depth_loss_w > 0 needs each ray's target depth: step(..., depth=...)")
        if depth is not None and self.depth_w == 0:
            raise ValueError("depth is read by the depth loss only (StaticTrainStep(depth_loss_w=...))")
        if depth is not None:
            self.depth_gt.copy_(depth, non_blocking=True)
        if self.ext is None and self.intr is None:
            self.rays_o.copy_(rays_o, non_blocking=True)
            self.rays_d.copy_(rays_d, non_blocking=True)
        self.gt.copy_(rgb_gt, non_blocking=True)
        if alpha is not None and not self.random_bg:
            raise ValueError("alpha is read by the random background only (StaticTrainStep(random_bg=True))")
        if self.random_bg:
            if alpha is None:
                self.alpha.fill_(1.0)
            else:
                self.alpha.copy_(alpha, non_blocking=True)
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
        if self.tr.p2p is not None:
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
                self.enc.adopt_shadow(self.tr._shadow)
        self.tr.sync_master()   # peer-memory step: the fp32 master table is complete again on every rank

    def _finish_step(self):
        self.tr.step_count += 1
        if self.tr._shadow is not None:
            self.enc.adopt_shadow(self.tr._shadow)
        return self.loss_sum / (3.0 * self.n)

    def attach_ray_source(self, image_bank, poses, directions, seed: int = 0, fixed_img: int = -1):
        """Keep the training set resident (as the reference's ``train_dataset.to(device)``) and let the step draw
        its own batch: ``step_sampled()`` then needs no per-step input at all.  With several ranks pass a
        different ``seed`` per rank."""
        if self.random_bg:
            raise _lib.NgpError("the device-sampled step does not support random_bg yet; use step()")
        if self.depth_w > 0:
            raise _lib.NgpError("the device-sampled step does not support depth supervision yet; use step(depth=...)")
        if self.ext is not None:
            raise _lib.NgpError("the device-sampled step does not support extrinsics refinement yet; use "
                                "step(directions=..., img_idxs=...)")
        if self.intr is not None:
            raise _lib.NgpError("the device-sampled step does not support intrinsics refinement; use "
                                "step(img_idxs=..., pix_idxs=...)")
        f = lambda t: t.detach().to(self.dev, torch.float32).contiguous()  # noqa: E731
        bank, poses, directions = f(image_bank), f(poses), f(directions)
        if bank.ndim != 3 or bank.shape[0] != poses.shape[0] or bank.shape[1] != directions.shape[0] or bank.shape[2] < 3:
            raise ValueError(f"image bank {tuple(bank.shape)} vs {poses.shape[0]} poses x {directions.shape[0]} pixels")
        if self.em is not None and (self.em.n_img != bank.shape[0] or self.em.W * self.em.H != bank.shape[1]
                                    or int(fixed_img) >= 0):
            raise ValueError(f"the error map covers {self.em.n_img} images of {self.em.W}x{self.em.H} pixels, all "
                             f"drawn; the image bank is {tuple(bank.shape)}" + (f", fixed_img {fixed_img}"
                                                                                if int(fixed_img) >= 0 else ""))
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
