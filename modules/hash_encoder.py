"""fp32 multiresolution hash-grid encoder — mirrors modules/hash_encoder.py of the reference
(HashEncoder :147-285).  The table is one flat fp32 Parameter of L-level (offset, size) slabs."""
from __future__ import annotations

import ctypes

import torch

from taichi_nerfs_b200 import ops
from taichi_nerfs_b200.layout import make_hash_layout

torch_type = torch.float32


class _HashEncode(torch.autograd.Function):
    """forward(positions [N,3] in [0,1], table) -> [N, L*F].  backward: dL/dtable always; dL/dx only
    when the positions require grad (the reference returns None there, hash_encoder.py:277)."""

    @staticmethod
    def forward(ctx, positions, table, encoder):
        out = ops.hash_encode_fwd(positions, table, encoder._clayout, encoder.out_dim)
        ctx.encoder = encoder
        ctx.save_for_backward(positions, table)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        positions, table = ctx.saved_tensors
        enc = ctx.encoder
        dy = grad_out.to(table.dtype).contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.hash_encode_bwd_input(positions, table, dy, enc._clayout)
        if enc.grad_sink is not None:
            # fused-optimizer path: accumulate straight into the trainer's flat gradient buffer
            ops.hash_encode_bwd(positions, dy, enc._clayout, enc.grad_sink)
            return dx, None, None
        grad_table = torch.zeros(table.numel(), device=table.device, dtype=torch.float32)
        ops.hash_encode_bwd(positions, dy, enc._clayout, grad_table)
        return dx, grad_table.view_as(table), None


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

        self.hash_table = torch.nn.Parameter(self._init_table(lay), requires_grad=True)
        self.grad_sink = None  # optional fp32 [P] buffer the backward accumulates into

    @staticmethod
    def _init_table(lay):
        # reference: flat table, U[0,1) (hash_encoder.py:220-227)
        return torch.rand(lay.total_param_size, dtype=torch.float32)

    def forward(self, positions):
        return _HashEncode.apply(positions.float().contiguous(), self.hash_table.contiguous(), self)

    # ---- kernel-level interface (NGP's grid update and the frame renderers) -------------------------------------
    emb_dtype = torch.float32

    def kernel_table(self):
        """The tensor the encode kernel reads (its pointer is tracked by FrameRenderer's graph)."""
        return self.hash_table.detach().contiguous()

    def encode_world(self, xyzs_w, aabb):
        """[N, out_dim] embedding of world positions, aabb = (xyz_min[3], xyz_max-xyz_min[3]) normalised in the
        kernel; no autograd."""
        return ops.hash_encode_fwd(xyzs_w, self.kernel_table(), self._clayout, self.out_dim, aabb=aabb)

    def enqueue_encode_dyn(self, lib, xyzs, table, emb, n_max, n_dev, aabb6, stream):
        """Raw launch of the device-counted encode (FrameRenderer's rounds): pointers in, rc out."""
        return lib.ngp_hash_encode_fwd_dyn(xyzs, table, ctypes.byref(self._clayout), emb, ops.F32, n_max, n_dev, aabb6,
                                           stream)
