"""fp32 multiresolution hash-grid encoder — mirrors modules/hash_encoder.py of the reference
(HashEncoder :147-285).  The table is one flat fp32 Parameter of L-level (offset, size) slabs.  The fp16 encoder
(``--half_opt``, modules/hash_encoder_half.py) is a subclass that changes the table and its precision only."""
from __future__ import annotations

import ctypes
import sys

import torch

from taichi_nerfs_b200 import ops
from taichi_nerfs_b200.layout import make_hash_layout

torch_type = torch.float32


class _HashEncode(torch.autograd.Function):
    """forward(positions [N,3] in [0,1], table, encoder) -> [N, L*F] of the encoder's emb_dtype, gathered from
    encoder.kernel_table().  backward: dL/dtable always; dL/dx only when the positions require grad (the reference
    returns None there, hash_encoder.py:277)."""

    @staticmethod
    def forward(ctx, positions, table, encoder):
        out = ops.hash_encode_fwd(positions, encoder.kernel_table(), encoder._clayout, encoder.out_dim)
        ctx.encoder = encoder
        ctx.save_for_backward(positions, table)   # (the table too: autograd refuses it if modified in place since)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        positions, _ = ctx.saved_tensors
        enc = ctx.encoder
        dy = grad_out.to(enc.emb_dtype).contiguous()
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.hash_encode_bwd_input(positions, enc.kernel_table(), dy, enc._clayout)
        if enc.grad_sink is not None:
            # fused-optimizer path: accumulate straight into the trainer's flat gradient buffer
            ops.hash_encode_bwd(positions, dy, enc._clayout, enc.grad_sink)
            return dx, None, None
        grad_table = enc._zeroed_table_grad()
        ops.hash_encode_bwd(positions, dy, enc._clayout, grad_table)
        return dx, grad_table, None


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

        print(f'Hash Encoder: base_res={base_res} max_res={max_res} hash_level={levels} '
              f'feat_per_level={feature_per_level} per_level_scale={self.log_b} '
              f'total_hash_size={lay.total_entries} ', file=sys.stderr)

        self._init_table(lay)
        self.grad_sink = None  # optional fp32 [P] buffer the backward accumulates into

    def _init_table(self, lay):
        # reference: flat table, U[0,1) (hash_encoder.py:220-227)
        self.hash_table = torch.nn.Parameter(torch.rand(lay.total_param_size, dtype=torch.float32), requires_grad=True)

    def _zeroed_table_grad(self):
        """The zeroed fp32 buffer, of the table's shape, that a backward without grad_sink accumulates into and
        returns."""
        return torch.zeros_like(self.hash_table, dtype=torch.float32)

    def forward(self, positions):
        return _HashEncode.apply(positions.float().contiguous(), self.hash_table, self)

    # ---- kernel-level interface (NGP's grid update, the frame renderers and the graph-captured step) --------------
    emb_dtype = torch.float32

    @property
    def bwd_raises_inf(self):
        """Whether the table backward raises GradScaler's inf flag itself (its F = 2 instantiation does)."""
        return self._clayout.feat_dim == 2

    def kernel_table(self):
        """The tensor the encode kernel reads (its pointer is tracked by FrameRenderer's graph)."""
        return self.hash_table.detach().contiguous()

    def encode_world(self, xyzs_w, aabb):
        """[N, out_dim] embedding of world positions, aabb = (xyz_min[3], xyz_max-xyz_min[3]) normalised in the
        kernel; no autograd."""
        return ops.hash_encode_fwd(xyzs_w, self.kernel_table(), self._clayout, self.out_dim, aabb=aabb)

    def _tag(self):
        return ops.F16 if self.emb_dtype == torch.float16 else ops.F32

    def enqueue_encode_dyn(self, lib, xyzs, table, emb, n_max, n_dev, aabb6, stream):
        """Raw launch of the device-counted encode (FrameRenderer's rounds, the graph-captured step): pointers in,
        rc out."""
        return lib.ngp_hash_encode_fwd_dyn(xyzs, table, ctypes.byref(self._clayout), emb, self._tag(), n_max, n_dev,
                                           aabb6, stream)

    def enqueue_encode_bwd_dyn(self, lib, xyzs, table, demb, grad_table, n_max, n_dev, aabb6, found_inf, stream):
        """Raw launch of the device-counted table backward (the graph-captured step) over all levels: grad_table +=
        dL/dtable of the first min(n_max, *n_dev) rows; found_inf (may be None) is raised on a non-finite
        contribution when bwd_raises_inf.  The table is not read: the hash gradient does not depend on it."""
        return lib.ngp_hash_encode_bwd_levels(xyzs, demb, self._tag(), ctypes.byref(self._clayout), grad_table, n_max,
                                              n_dev, aabb6, 0, self._clayout.n_levels, found_inf, stream)
