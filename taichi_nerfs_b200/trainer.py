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
                 p2p_optimizer: bool | None = None, voxel_reg=None):
        # voxel_reg = (w_tv_sigma, w_tv_sh, w_sparsity): the voxel grid's regularisers (DESIGN.md §6d), enqueued after
        # the render backward.  None or all zero: nothing is enqueued.
        self.voxel_reg = None
        if voxel_reg is not None:
            if not (hasattr(model, 'sh_fields') and hasattr(model, 'density_fields')):
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

        self.params = [p for p in model.parameters() if p.requires_grad]
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
        # a model without a position encoder (VoxelGrid) scatters into the .grad views of its own parameters
        P_, enc_ = sizes[0], getattr(model, 'pos_encoder', None)
        if p2p_optimizer and (enc_ is None or hasattr(enc_, 'plane_embedding')):
            raise ValueError("NGPTrainer: the peer-memory optimizer shards the fp16 hash table; a tri-plane or "
                             "voxel-grid model uses the all-reduce of the flat gradient (p2p_optimizer off)")
        if (p2p_optimizer is not False and self.world_size > 1 and dev.type == "cuda" and hasattr(enc_, "adopt_shadow")
                and self.params[0] is enc_.hash_table and P_ % (4 * self.world_size) == 0):
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
            if enc_ is not None and (p is getattr(enc_, 'hash_table', None)
                                     or p is getattr(enc_, 'plane_embedding', None)):
                enc_.grad_sink = self.flat_grad[off - s - q:off - q]
        if enc_ is None:
            model.grad_sink = (model.sh_fields.grad, model.density_fields.grad)
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
        enc = enc_
        if hasattr(enc, "adopt_shadow"):
            assert self.params[0] is enc.hash_table, "the hash table must be the first parameter"
            # fp16 copy of the whole flat buffer, rewritten by the Adam pass; the encoder reads its first slice
            if self.p2p is not None:
                self._shadow_full = self.p2p.shadow
                self._shadow_full.copy_(self.flat_param)
            else:
                self._shadow_full = self.flat_param.to(torch.float16)
            self._shadow = self._shadow_full[:enc.hash_table.numel()]
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
        enc = getattr(self.model, 'pos_encoder', self.model)   # a VoxelGrid holds its grad_sink itself
        if hasattr(enc, 'grad_sink'):
            enc.grad_sink = None
        if self._shadow is not None and hasattr(enc, 'adopt_shadow'):
            enc.adopt_shadow(None)
        self._views = []

    def forward_backward(self, rays_o, rays_d, rgb_gt, exp_step_factor=0.0, extra_loss=None):
        from modules.rendering import render
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            results = render(self.model, rays_o, rays_d, exp_step_factor=exp_step_factor)
            loss = F.mse_loss(results['rgb'], rgb_gt)
            if extra_loss is not None:  # e.g. distortion loss (train.py:194-195)
                loss = loss + extra_loss(results)
        # GradScaler.scale(loss): the current scale is a device scalar, no host read
        scale = self.scale_state[0] if self.dynamic_loss_scale else self.loss_scale
        (loss * scale).backward()
        if self.voxel_reg is not None:
            self.add_voxel_reg()
        return loss, results

    def add_voxel_reg(self, loss=None):
        """Add loss_scale * the gradient of the voxel regularisers into the flat gradient (the model's grad_sink), from
        the parameters the forward read; the scale is the device value when it is dynamic.  loss (fp32 [1], optional)
        accumulates the unscaled weighted regulariser loss."""
        m = self.model
        dsh, dden = m.grad_sink
        dyn = self.scale_state if self.dynamic_loss_scale else None
        ops.voxel_reg(m.sh_fields.detach(), m.density_fields.detach(), m._clayout, m._reg_block, self.voxel_reg, dsh,
                      dden, loss_scale=self.loss_scale, scale_dev=dyn, loss=loss)

    def enqueue_update(self, check_finite: bool = True):
        """Gradient exchange -> inf check -> LR / bias-correction scalars -> fused Adam (+fp16 shadow, grad zero) ->
        GradScaler.update(), all on the current stream with device-side scalars (graph-capturable).

        The exchange: none on one rank.  Peer memory (csrc/p2p.cu): [local finite check] -> barrier (all backward
        passes done; found_inf becomes the OR over the ranks) -> ONE kernel: peer-load sum of the owned gradient slice +
        Adam on it + peer-store of the new fp16 table slice into every rank's shadow (the MLP weights: every rank, same
        sums) -> barrier (everybody has read my gradient and written my shadow) -> clear the local gradient.  NCCL
        fallback: pack the gradient to fp16 -> ONE all-reduce of half the bytes -> finite check on the reduced buffer
        (always: identical on every rank, catches local inf/NaN and overflow alike) -> Adam reads the fp16 sum and
        zeroes the fp32 accumulation buffer.

        check_finite=False: the backward kernels already raised the inf flag at the source (fast_step.py)."""
        L, st = load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
        R, fg, g16, P = self.p2p, self.flat_grad, self.grad16, self.slices[0][1]
        if g16 is not None:
            check(L.ngp_grad_pack_f16(_p(fg), _p(g16), fg.numel(), st))
            parallel.allreduce_gradients(g16, self.pg)
            check(L.ngp_check_finite_f16(_p(g16), g16.numel(), _p(self.found_inf), st))
        elif check_finite:
            check(L.ngp_check_finite(_p(fg), fg.numel(), _p(self.found_inf), st))
        if R is not None:
            R.barrier(self.found_inf)
        # inv_scale: static (host constant) or the device value maintained by GradScaler.update() below (-1 sentinel)
        inv = -1.0 if self.dynamic_loss_scale else parallel.inv_grad_scale(self.loss_scale, self.world_size)
        check(L.ngp_adam_hyper_update(_p(self.step_dev), self.lr0, self.lr0 / 30, self.max_steps, self.betas[0],
                                      self.betas[1], inv, _p(self.found_inf), _p(self.hyper), st))
        # one Adam launch over [hash table | MLP weights]
        if R is not None:
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
        self.enqueue_update()
        if self._shadow is not None:
            self.model.pos_encoder.adopt_shadow(self._shadow)

    def step(self, rays_o, rays_d, rgb_gt, exp_step_factor=0.0, extra_loss=None):
        loss, results = self.forward_backward(rays_o, rays_d, rgb_gt, exp_step_factor, extra_loss)
        self.optimizer_step()
        return loss, results
