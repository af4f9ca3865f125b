"""fp16 multiresolution hash-grid encoder (``--half_opt``) — mirrors
modules/hash_encoder_half.py of the reference (HashEncoder :218-368): fp32 master table of shape
[entries, F], gathers from an fp16 copy with fp16 accumulation, fp32 gradient accumulation."""
from __future__ import annotations

import ctypes

import torch

from taichi_nerfs_b200 import ops
from taichi_nerfs_b200.layout import make_hash_layout

torch_type = torch.float16


class _HashEncodeHalf(torch.autograd.Function):

    @staticmethod
    def forward(ctx, positions, table_f32, encoder):
        shadow = encoder.table_f16()
        out = ops.hash_encode_fwd(positions, shadow, encoder._clayout, encoder.out_dim)
        ctx.encoder = encoder
        ctx.save_for_backward(positions)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        positions, = ctx.saved_tensors
        enc = ctx.encoder
        # the reference zeroes its persistent `hash_grad` buffer and accumulates into it
        # (hash_encoder_half.py:350-361)
        dy = grad_out.to(torch.float16).contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.hash_encode_bwd_input(positions, enc.table_f16(), dy, enc._clayout)
        if enc.grad_sink is not None:
            # fused-optimizer path: accumulate straight into the trainer's flat gradient buffer
            ops.hash_encode_bwd(positions, dy, enc._clayout, enc.grad_sink)
            return dx, None, None
        hash_grad = enc.hash_grad.zero_()
        ops.hash_encode_bwd(positions, dy, enc._clayout, hash_grad)
        return dx, hash_grad, None


class HashEncoder(torch.nn.Module):

    def __init__(self, max_params: float = 2 ** 19, levels: int = 16, base_res: float = 16.0,
                 max_res: float = 2048.0, feature_per_level: int = 2):
        super().__init__()
        lay = make_hash_layout(max_params, levels, base_res, max_res, feature_per_level)
        self._layout = lay
        self._clayout = lay.as_ctypes()
        self.log_b = lay.log_b
        self.base_res = base_res
        self.hash_level = levels
        self.max_params = max_params
        self.feature_per_level = feature_per_level
        self.out_dim = lay.out_dim
        self.begin_fast_hash_level = lay.begin_fast_hash_level
        self.total_param_size = lay.total_param_size

        self.register_buffer('offsets', torch.tensor(lay.offsets, dtype=torch.int32), persistent=False)
        self.register_buffer('hash_map_sizes', torch.tensor(lay.map_sizes, dtype=torch.int32), persistent=False)

        import sys
        print(f'Hash Encoder: base_res={base_res} max_res={max_res} hash_level={levels} '
              f'feat_per_level={feature_per_level} per_level_scale={self.log_b} '
              f'total_hash_size={lay.total_entries} ', file=sys.stderr)

        # fp32 master [entries, F], U(-1e-4, 1e-4) (hash_encoder_half.py:291-299)
        table = (torch.rand(lay.total_entries, feature_per_level, dtype=torch.float32) * 2.0 - 1.0) * 1e-4
        self.hash_table = torch.nn.Parameter(table, requires_grad=True)
        self.register_buffer('hash_grad', torch.zeros_like(table, dtype=torch.float32))
        # fp16 shadow of the master: refreshed lazily (or written directly by the fused Adam pass)
        self._shadow = None
        self._shadow_version = -1
        self.grad_sink = None  # optional fp32 [entries*F] buffer the backward accumulates into

    def table_f16(self):
        """fp16 copy of the table used by the kernels.  The reference re-casts on every forward
        (hash_encoder_half.py:367); here the cast is skipped while the master is unchanged."""
        p = self.hash_table
        if (self._shadow is None or self._shadow.device != p.device or self._shadow_version != p._version):
            self._shadow = p.detach().to(torch.float16).contiguous()
            self._shadow_version = p._version
        return self._shadow

    def adopt_shadow(self, shadow):
        """Called by the fused optimizer after it rewrote master + fp16 shadow in one pass."""
        self._shadow = shadow
        self._shadow_version = self.hash_table._version

    def forward(self, positions):
        out = _HashEncodeHalf.apply(positions.float().contiguous(), self.hash_table, self)
        return out.view(-1, self.out_dim)

    # ---- kernel-level interface (NGP's grid update and the frame renderers) -------------------------------------
    emb_dtype = torch.float16

    def kernel_table(self):
        """The tensor the encode kernel reads (its pointer is tracked by FrameRenderer's graph)."""
        return self.table_f16()

    def encode_world(self, xyzs_w, aabb):
        """[N, out_dim] embedding of world positions, aabb = (xyz_min[3], xyz_max-xyz_min[3]) normalised in the
        kernel; no autograd."""
        return ops.hash_encode_fwd(xyzs_w, self.kernel_table(), self._clayout, self.out_dim, aabb=aabb)

    def enqueue_encode_dyn(self, lib, xyzs, table, emb, n_max, n_dev, aabb6, stream):
        """Raw launch of the device-counted encode (FrameRenderer's rounds): pointers in, rc out."""
        return lib.ngp_hash_encode_fwd_dyn(xyzs, table, ctypes.byref(self._clayout), emb, ops.F16, n_max, n_dev, aabb6,
                                           stream)
