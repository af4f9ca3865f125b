"""Training step of the NGP hot path (the body of the reference's loop, train.py:168-201):
get_rays -> render -> MSE -> backward -> [gradient all-reduce] -> optimizer step.

``NGPTrainer.step`` keeps the reference's numerics (torch.autocast(fp16), GradScaler(2**16 | 2**19) with its
dynamic scale: x0.5 on inf/NaN, x2 every 2000 clean steps, skipped steps do not advance Adam's step count;
Adam(eps=1e-15), cosine LR to lr/30) but replaces optimizer.zero_grad + GradScaler.unscale_/inf-check + Adam +
the fp16 table re-cast by ONE fused pass over the flat parameter buffer (csrc/optim.cu).  The scale, the LR /
bias-correction scalars and the iteration counter live in device memory (``scale_state``, ``hyper``, ``step_dev``),
so nothing synchronises the host; the graph-captured step (fast_step.py) enqueues exactly the same kernels.

Multi-GPU: rays are sharded across ranks (each rank renders its own batch) and the gradient sum is folded into the
fused Adam as inv_scale / world_size (SURVEY.md §8e).  On one NVLink box the optimizer step is ONE peer-memory kernel
(csrc/p2p.cu); otherwise the flat gradient is all-reduced once per step in fp16 over NCCL.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn.functional as F

from . import ops, parallel
from ._lib import check, load


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class NGPTrainer:
    def __init__(self, model, lr: float = 1e-2, max_steps: int = 20000, loss_scale: float | None = None,
                 betas=(0.9, 0.999), eps: float = 1e-15, process_group=None, dynamic_loss_scale: bool = True,
                 p2p_optimizer: bool | None = None, voxel_reg=None, extrinsics=None, exposure=None,
                 intrinsics=None):
        from modules.hash_encoder import HashEncoder
        from modules.voxel_grid import VoxelGrid
        from .exposure import ExposureCorrection
        from .extrinsics import PoseRefinement
        from .intrinsics import IntrinsicsRefinement
        # The model kind, decided here once (StaticTrainStep reads it too): the position encoder, whose one parameter
        # (its table) must be the first slice of the flat buffers, or None for a VoxelGrid, which has no encoder and
        # scatters into the .grad views of its own fields.
        self.encoder = enc = None if isinstance(model, VoxelGrid) else model.pos_encoder
        # voxel_reg = (w_tv_sigma, w_tv_sh, w_sparsity): the voxel grid's regularisers (DESIGN.md §6d), enqueued after
        # the render backward.  None or all zero: nothing is enqueued.
        self.voxel_reg = None
        if voxel_reg is not None:
            if enc is not None:
                raise ValueError("NGPTrainer: voxel_reg (total variation / sparsity) applies to a model with voxel "
                                 "fields (--model_name svox); this model has none")
            w = tuple(float(v) for v in voxel_reg)
            if len(w) != 3 or not all(math.isfinite(v) and v >= 0 for v in w):
                raise ValueError(f"NGPTrainer: voxel_reg must be three finite weights >= 0 "
                                 f"(w_tv_sigma, w_tv_sh, w_sparsity), got {voxel_reg}")
            self.voxel_reg = w if any(w) else None
        self.model = model
        self.lr0 = lr
        self.max_steps = max_steps
        self.betas = betas
        self.eps = eps
        # train.py:137-141: GradScaler(2**16) with --half_opt, else 2**19
        self.loss_scale = float(loss_scale if loss_scale is not None else (2 ** 16 if model.half_opt else 2 ** 19))
        self.step_count = 0
        self.pg = process_group
        self.world_size = 1
        if process_group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            self.world_size = torch.distributed.get_world_size(process_group)

        # camera extrinsics refinement (DESIGN.md §6i): a PoseRefinement whose Adam step runs with the model's, or None
        if extrinsics is not None:
            if not isinstance(extrinsics, PoseRefinement):
                raise TypeError("NGPTrainer: extrinsics must be a taichi_nerfs_b200.extrinsics.PoseRefinement")
            if not isinstance(enc, HashEncoder):
                raise ValueError("NGPTrainer: extrinsics refinement needs the gradient wrt the sample positions, which "
                                 "only the hash encoder provides (not the tri-plane encoder or the voxel grid)")
            if self.world_size > 1:
                raise ValueError("NGPTrainer: extrinsics refinement runs on one rank (the pose gradient is not "
                                 "exchanged between ranks)")
        self.extrinsics = extrinsics
        # camera intrinsics refinement (DESIGN.md §6l): an IntrinsicsRefinement whose Adam step runs with the model's
        if intrinsics is not None:
            if not isinstance(intrinsics, IntrinsicsRefinement):
                raise TypeError("NGPTrainer: intrinsics must be a taichi_nerfs_b200.intrinsics.IntrinsicsRefinement")
            if not isinstance(enc, HashEncoder):
                raise ValueError("NGPTrainer: intrinsics refinement needs the gradient wrt the sample positions, which "
                                 "only the hash encoder provides (not the tri-plane encoder or the voxel grid)")
            if self.world_size > 1:
                raise ValueError("NGPTrainer: intrinsics refinement runs on one rank (its gradient is not exchanged "
                                 "between ranks)")
        self.intrinsics = intrinsics
        # per-image exposure compensation (DESIGN.md §6k): an ExposureCorrection whose Adam step runs with the model's
        if exposure is not None:
            if not isinstance(exposure, ExposureCorrection):
                raise TypeError("NGPTrainer: exposure must be a taichi_nerfs_b200.exposure.ExposureCorrection")
            if self.world_size > 1:
                raise ValueError("NGPTrainer: exposure compensation runs on one rank (the exposure gradient is not "
                                 "exchanged between ranks)")
        self.exposure = exposure
        self._pose_batch = None   # (xyzs, ts, rays_a, img_idxs, rays_d) of the last forward_backward

        self.params = [p for p in model.parameters() if p.requires_grad]
        if enc is not None:
            table = list(enc.parameters())
            if len(table) != 1 or table[0] is not self.params[0]:
                raise ValueError("NGPTrainer: the position encoder must have one parameter, the model's first")
        # the fp16 hash encoder gathers from an fp16 copy of its table, which the fused Adam rewrites (the shadow below)
        shadowed = enc is not None and enc.emb_dtype == torch.float16
        dev = self.params[0].device
        # one flat gradient buffer so the multi-GPU path is a single all-reduce (hash grad | MLP grads)
        sizes = [p.numel() for p in self.params]
        pad = [(-s) % 4 for s in sizes]  # keep every slice 16-byte aligned for the float4 Adam kernel
        total = sum(s + q for s, q in zip(sizes, pad))
        # Several ranks on one NVLink box (p2p_optimizer: None = whenever available, False = the NCCL fallback): the
        # gradient and the fp16 shadow live in a CUDA-IPC buffer that the peers map, and the optimizer step is ONE
        # kernel that sums the owned 1/N of the gradient with peer loads, runs Adam on it and stores the new fp16 table
        # slice into every rank's shadow with peer stores (csrc/p2p.cu).  None when unavailable (NCCL fallback below).
        self.p2p = None
        P_ = sizes[0]
        if p2p_optimizer and not isinstance(enc, HashEncoder):
            raise ValueError("NGPTrainer: the peer-memory optimizer shards the fp16 hash table; a tri-plane or "
                             "voxel-grid model uses the all-reduce of the flat gradient (p2p_optimizer off)")
        if (p2p_optimizer is not False and self.world_size > 1 and dev.type == "cuda" and shadowed
                and P_ % (4 * self.world_size) == 0):
            from .p2p import PeerRegion
            self.p2p = PeerRegion.create(total, dev, process_group)
        self.flat_grad = self.p2p.grad if self.p2p is not None else torch.zeros(total, device=dev, dtype=torch.float32)
        # parameters live in one flat buffer as well (each nn.Parameter becomes a view of it, state_dict is
        # unchanged), so the fused Adam is ONE launch over [hash table | MLP weights]
        self.flat_param = torch.zeros(total, device=dev, dtype=torch.float32)
        self.exp_avg = torch.zeros(total, device=dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(total, device=dev, dtype=torch.float32)
        self.slices = []
        off = 0
        for p, s, q in zip(self.params, sizes, pad):
            self.slices.append((off, s))
            p.grad = self.flat_grad[off:off + s].view_as(p)  # autograd accumulates straight into the flat buffer
            with torch.no_grad():
                self.flat_param[off:off + s].copy_(p.data.reshape(-1))
            p.data = self.flat_param[off:off + s].view_as(p)
            off += s + q
        if enc is None:
            model.grad_sink = (model.sh_fields.grad, model.density_fields.grad)
        else:
            enc.grad_sink = self.flat_grad[:P_]
        self.found_inf = torch.zeros(1, device=dev, dtype=torch.int32)
        # device-side optimizer scalars (shared with StaticTrainStep): iteration counter, [lr/bc1, sqrt(bc2), 1/(scale*world),
        # Adam step count], GradScaler state [scale, growth tracker]
        self.dynamic_loss_scale = bool(dynamic_loss_scale)
        self.step_dev = torch.zeros(1, device=dev, dtype=torch.int32)
        self.hyper = torch.zeros(4, device=dev, dtype=torch.float32)
        self.hyper[2] = parallel.inv_grad_scale(self.loss_scale, self.world_size)
        self.scale_state = torch.tensor([self.loss_scale, 0.0], device=dev, dtype=torch.float32)
        self._views = [(p, p.data_ptr(), p.grad.data_ptr()) for p in self.params]
        self._shadow = self._shadow_full = None
        if shadowed:
            # fp16 copy of the whole flat buffer, rewritten by the Adam pass; the encoder reads its first slice
            if self.p2p is not None:
                self._shadow_full = self.p2p.shadow
                self._shadow_full.copy_(self.flat_param)
            else:
                self._shadow_full = self.flat_param.to(torch.float16)
            self._shadow = self._shadow_full[:P_]
            enc.adopt_shadow(self._shadow)

        # Peer-memory step: the optimizer is sharded over the hash table (the MLP weights stay replicated); each rank
        # owns 1/N of the table.  The fp32 master of non-owned entries goes stale until sync_master() (called before
        # state_dict / checkpoints).
        if self.p2p is not None:
            self.rank = torch.distributed.get_rank(process_group)
            self.shard_lo, hi = parallel.optimizer_shard(P_, self.rank, self.world_size)
            self.shard = hi - self.shard_lo
            self.master_stale = False
        # Several ranks without peer memory: the gradient travels in fp16 (half the all-reduce bytes).  That is the
        # precision the reference's own gradients have under autocast (fp16 autograd); the loss scale keeps them in
        # range and an overflow becomes inf = a skipped step + scale backoff, as with GradScaler.
        self.grad16 = (torch.zeros(total, device=dev, dtype=torch.float16)
                       if self.world_size > 1 and self.p2p is None else None)

    # cosine annealing to lr/30 (train.py:159-163, CosineAnnealingLR(T_max=max_steps, eta_min=lr/30))
    def lr_at(self, step: int) -> float:
        eta_min = self.lr0 / 30
        return eta_min + (self.lr0 - eta_min) * (1 + math.cos(math.pi * min(step, self.max_steps) / self.max_steps)) / 2

    def check_aliasing(self):
        """The fused optimizer updates parameters through the flat buffers: every nn.Parameter must still be the view
        created in __init__ (model.to()/half(), zero_grad(set_to_none=True) or a foreign optimizer break that)."""
        for p, dptr, gptr in self._views:
            if p.data_ptr() != dptr or p.grad is None or p.grad.data_ptr() != gptr:
                raise RuntimeError("NGPTrainer: a parameter or its .grad no longer aliases the flat buffers (was the "
                                   "model moved / cast, or its gradients set to None?) — build a new NGPTrainer")

    def detach(self):
        """Give the model ordinary, independent parameters again (e.g. before handing it to a torch optimizer)."""
        for p in self.params:
            p.data = p.data.clone()
            p.grad = None
        if self.encoder is None:   # a VoxelGrid holds its grad_sink itself
            self.model.grad_sink = None
        else:
            self.encoder.grad_sink = None
        if self._shadow is not None:
            self.encoder.adopt_shadow(None)
        self._views = []

    def forward_backward(self, rays_o, rays_d, rgb_gt, exp_step_factor=0.0, extra_loss=None, bg_rgb=None, alpha=None,
                         b_load=1.0, img_idxs=None, ray_w=None, pix_idxs=None):
        """bg_rgb [N, 3] (--random_bg, ops.random_bg): each ray's background colour replaces the fixed one; with
        ``alpha`` [N] (the image's alpha), the target's loader background ``b_load`` is replaced by it too:
        rgb_gt + (bg_rgb - b_load)(1 - alpha).  With extrinsics refinement, ``img_idxs`` [N] (or one index) names each
        ray's image and rays_o / rays_d are the PoseRefinement's rays; the pose gradient is formed by optimizer_step.
        With exposure compensation, ``img_idxs`` names each ray's image too, and the sample colours pass through its
        gain (DESIGN.md §6k).
        With intrinsics refinement (DESIGN.md §6l) the rays' camera directions are the IntrinsicsRefinement's
        ``directions(pix_idxs)``; ``pix_idxs`` [N] and ``img_idxs`` are required, and the intrinsics gradient is formed
        by optimizer_step.
        ``ray_w`` [N] fp32 (error-map sampling, DESIGN.md §6j): the MSE becomes mean_r w_r mean_c (rgb - gt)^2, and the
        returned loss is that weighted value; ``extra_loss`` weights its own per-ray terms."""
        from modules.rendering import render
        intr = self.intrinsics
        refine = self.extrinsics is not None or intr is not None
        expo = self.exposure
        if refine and img_idxs is None:
            raise ValueError("NGPTrainer: camera refinement needs each ray's image index (img_idxs=...)")
        if intr is not None:
            if pix_idxs is None or intr.pix is None or intr.n_rays != len(rays_o):
                raise ValueError("NGPTrainer: intrinsics refinement needs each ray's pixel (pix_idxs=...), with the "
                                 "directions of IntrinsicsRefinement.directions(pix_idxs) of this batch")
        elif pix_idxs is not None:
            raise ValueError("NGPTrainer: pix_idxs is read by intrinsics refinement only (NGPTrainer(intrinsics=...))")
        if expo is not None and img_idxs is None:
            raise ValueError("NGPTrainer: exposure compensation needs each ray's image index (img_idxs=...)")
        if not refine and expo is None and img_idxs is not None:
            raise ValueError("NGPTrainer: img_idxs is read by camera refinement and exposure compensation only "
                             "(NGPTrainer(extrinsics=... | intrinsics=... | exposure=...))")
        exposure = None if expo is None else (lambda rgbs, rays_a: expo.apply(rgbs, rays_a, img_idxs))  # noqa: E731
        if bg_rgb is not None and alpha is not None:
            rgb_gt = rgb_gt + (bg_rgb - b_load) * (1 - alpha)[:, None]
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            results = render(self.model, rays_o, rays_d, exp_step_factor=exp_step_factor, bg_rgb=bg_rgb,
                             position_grad=refine, exposure=exposure)
            if ray_w is None:
                loss = F.mse_loss(results['rgb'], rgb_gt)
            else:
                loss = ((results['rgb'].float() - rgb_gt) ** 2).mean(-1).mul(ray_w).mean()
            if extra_loss is not None:  # e.g. distortion loss (train.py:194-195)
                loss = loss + extra_loss(results)
        # GradScaler.scale(loss): the current scale is a device scalar, no host read
        scale = self.scale_state[0] if self.dynamic_loss_scale else self.loss_scale
        (loss * scale).backward()
        if self.voxel_reg is not None:
            self.add_voxel_reg()
        if refine:
            self._pose_batch = (results.pop('xyzs'), results['ts'], results['rays_a'], img_idxs, rays_d)
        return loss, results

    def enqueue_pose_grad(self):
        """Camera refinement: the pose and intrinsics gradients of the last forward_backward (its sample positions'
        .grad) into the PoseRefinement's and IntrinsicsRefinement's buffers, raising found_inf on a non-finite
        contribution."""
        xyzs, ts, rays_a, img_idxs, rays_d = self._pose_batch
        self._pose_batch = None
        dx = xyzs.grad
        if dx is None:   # no sample reached the network
            return
        if self.extrinsics is not None:
            self.extrinsics.accumulate(dx, ts, rays_a, img_idxs, rays_d.float(), found_inf=self.found_inf)
        if self.intrinsics is not None:
            self.intrinsics.accumulate(dx.float(), ts, rays_a, img_idxs,
                                       pose_corr=None if self.extrinsics is None else self.extrinsics.corr,
                                       found_inf=self.found_inf)

    def add_voxel_reg(self, loss=None):
        """Add loss_scale * the gradient of the voxel regularisers into the flat gradient (the model's grad_sink), from
        the parameters the forward read; the scale is the device value when it is dynamic.  loss (fp32 [1], optional)
        accumulates the unscaled weighted regulariser loss."""
        m = self.model
        dsh, dden = m.grad_sink
        dyn = self.scale_state if self.dynamic_loss_scale else None
        ops.voxel_reg(m.sh_fields.detach(), m.density_fields.detach(), m._clayout, m._reg_block, self.voxel_reg, dsh,
                      dden, loss_scale=self.loss_scale, scale_dev=dyn, loss=loss)

    def voxel_fields(self):
        """(param, grad, exp_avg, exp_avg_sq) views [G, G, G, C] of the sh field and of the density field in the flat
        buffers, for the node-block optimizer pass (enqueue_update(voxel_block=...))."""
        out = []
        for p, (off, n) in zip(self.params, self.slices):
            out.append(tuple(t[off:off + n].view(p.shape) for t in (self.flat_param, self.flat_grad, self.exp_avg,
                                                                    self.exp_avg_sq)))
        return out

    def enqueue_update(self, check_finite: bool = True, voxel_block=None):
        """Gradient exchange -> inf check -> LR / bias-correction scalars -> fused Adam (+fp16 shadow, grad zero) ->
        GradScaler.update(), all on the current stream with device-side scalars (graph-capturable).

        The exchange: none on one rank.  Peer memory (csrc/p2p.cu): [local finite check] -> barrier (all backward
        passes done; found_inf becomes the OR over the ranks) -> ONE kernel: peer-load sum of the owned gradient slice +
        Adam on it + peer-store of the new fp16 table slice into every rank's shadow (the MLP weights: every rank, same
        sums) -> barrier (everybody has read my gradient and written my shadow) -> clear the local gradient.  NCCL
        fallback: pack the gradient to fp16 -> ONE all-reduce of half the bytes -> finite check on the reduced buffer
        (always: identical on every rank, catches local inf/NaN and overflow alike) -> Adam reads the fp16 sum and
        zeroes the fp32 accumulation buffer.

        check_finite=False: the backward kernels already raised the inf flag at the source (fast_step.py).

        voxel_block = (lo_x, lo_y, lo_z, hi_x, hi_y, hi_z), one rank, a voxel-grid model: the finite check and Adam run
        over the fields' elements inside that node block only (DESIGN.md §6b).  Elements outside it are neither checked,
        applied nor cleared, so the caller must know that its gradient is zero there, as StaticTrainStep does: every
        gradient its own march, backward and regularisers produce lies inside the block."""
        L, st = load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
        R, fg, g16, P = self.p2p, self.flat_grad, self.grad16, self.slices[0][1]
        if voxel_block is not None:
            if R is not None or g16 is not None or len(self.params) != 2:
                raise ValueError("NGPTrainer: the node-block optimizer pass is for a one-rank voxel-grid model")
            fields = self.voxel_fields()
            b6 = (C.c_int32 * 6)(*[int(v) for v in voxel_block])
        if voxel_block is not None and check_finite:
            for prm, grd, _, _ in fields:
                check(L.ngp_check_finite_voxel_block(_p(grd), prm.shape[0], prm.shape[-1], b6, _p(self.found_inf), st))
        elif g16 is not None:
            check(L.ngp_grad_pack_f16(_p(fg), _p(g16), fg.numel(), st))
            parallel.allreduce_gradients(g16, self.pg)
            check(L.ngp_check_finite_f16(_p(g16), g16.numel(), _p(self.found_inf), st))
        elif check_finite:
            check(L.ngp_check_finite(_p(fg), fg.numel(), _p(self.found_inf), st))
        if check_finite and self.exposure is not None:   # the exposure gradient is outside the flat buffer
            eg = self.exposure.grad
            check(L.ngp_check_finite(_p(eg), eg.numel(), _p(self.found_inf), st))
        if R is not None:
            R.barrier(self.found_inf)
        # inv_scale: static (host constant) or the device value maintained by GradScaler.update() below (-1 sentinel)
        inv = -1.0 if self.dynamic_loss_scale else parallel.inv_grad_scale(self.loss_scale, self.world_size)
        check(L.ngp_adam_hyper_update(_p(self.step_dev), self.lr0, self.lr0 / 30, self.max_steps, self.betas[0],
                                      self.betas[1], inv, _p(self.found_inf), _p(self.hyper), st))
        # one Adam launch over [hash table | MLP weights]
        if voxel_block is not None:   # one per field, over its node block
            for prm, grd, m, v in fields:
                check(L.ngp_adam_step_voxel_block_dyn(_p(prm), _p(grd), _p(m), _p(v), prm.shape[0], prm.shape[-1], b6,
                                                      _p(self.found_inf), _p(self.hyper), self.betas[0], self.betas[1],
                                                      self.eps, st))
        elif R is not None:
            check(L.ngp_adam_step_p2p(_p(self.flat_param), R.grad_tab, _p(self.exp_avg), _p(self.exp_avg_sq),
                                      R.shadow_tab, R.rank, R.world, _p(self.found_inf), _p(self.hyper), self.betas[0],
                                      self.betas[1], self.eps, self.shard_lo, self.shard_lo + self.shard, P,
                                      fg.numel(), st))
            R.barrier(None)
            fg.zero_()
            self.master_stale = True
        elif g16 is not None:
            check(L.ngp_adam_step_dyn_g16(_p(self.flat_param), _p(g16), _p(fg), _p(self.exp_avg), _p(self.exp_avg_sq),
                                          _p(self._shadow_full), _p(self.found_inf), _p(self.hyper), self.betas[0],
                                          self.betas[1], self.eps, fg.numel(), st))
        else:
            check(L.ngp_adam_step_dyn(_p(self.flat_param), _p(fg), _p(self.exp_avg), _p(self.exp_avg_sq),
                                      _p(self._shadow_full), _p(self.found_inf), _p(self.hyper), self.betas[0],
                                      self.betas[1], self.eps, 1, fg.numel(), st))
        if self.extrinsics is not None:   # the pose corrections' Adam, on the same device scalars (one rank)
            self.extrinsics.enqueue_adam(self)
        if self.exposure is not None:     # the exposures' Adam and zero-mean projection, on the same scalars
            self.exposure.enqueue_adam(self)
        if self.intrinsics is not None:   # the intrinsics corrections' reduction and Adam, on the same scalars
            self.intrinsics.enqueue_adam(self)
        if self.dynamic_loss_scale:  # GradScaler.update(): adjusts the scale used by the NEXT step
            # a flag raised at the source is not reset by the next step, so this launch clears it
            raised_at_source = not check_finite and g16 is None
            check(L.ngp_loss_scale_update(_p(self.scale_state), _p(self.found_inf), 2.0, 0.5, 2000,
                                          float(self.world_size), _p(self.hyper), int(raised_at_source), st))

    def p2p_check(self):
        """Host check (synchronises): raises if a peer barrier of this rank timed out (a rank fell out of step)."""
        if self.p2p is not None and self.p2p.timed_out():
            raise RuntimeError("NGPTrainer: a peer barrier timed out — the ranks did not run the same steps")

    def sync_master(self):
        """Peer-memory step: make the fp32 master table complete on every rank again (before state_dict(), checkpoints
        or anything else that reads ``hash_table`` itself rather than the fp16 shadow)."""
        if self.p2p is not None and self.master_stale:
            import torch.distributed as dist
            P, lo = self.slices[0][1], self.shard_lo
            own = self.flat_param[lo:lo + self.shard].clone()
            dist.all_gather_into_tensor(self.flat_param[:P], own, group=self.pg)
            self.master_stale = False

    def optimizer_step(self):
        self.check_aliasing()
        self.step_count += 1
        self.found_inf.zero_()
        if self.intrinsics is not None:   # pixels of the batch's directions() that were not invertible
            self.found_inf.copy_(self.intrinsics.flag)
            self.intrinsics.flag.zero_()
        if self._pose_batch is not None:
            self.enqueue_pose_grad()
        self.enqueue_update()
        if self._shadow is not None:
            self.encoder.adopt_shadow(self._shadow)

    def step(self, rays_o, rays_d, rgb_gt, exp_step_factor=0.0, extra_loss=None, bg_rgb=None, alpha=None, b_load=1.0,
             img_idxs=None, ray_w=None, pix_idxs=None):
        loss, results = self.forward_backward(rays_o, rays_d, rgb_gt, exp_step_factor, extra_loss, bg_rgb, alpha,
                                              b_load, img_idxs, ray_w, pix_idxs)
        self.optimizer_step()
        return loss, results
