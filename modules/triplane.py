"""Tri-plane position encoder — mirrors modules/triplane.py of the reference (TriPlaneEncoder :103-205): same
constructor, attributes (out_dim, log_b, total_param_size) and parameter (``plane_embedding``, flat fp32,
U[0,1) init).  The Taichi kernel and its autodiff are replaced by csrc/triplane.cu."""
from __future__ import annotations

import ctypes
import sys

import torch

from taichi_nerfs_b200 import ops
from taichi_nerfs_b200.layout import make_triplane_layout

torch_type = torch.float32


class _TriplaneEncode(torch.autograd.Function):
    """forward(positions [N,3] in [0,1], table) -> fp32 [N, L*F].  backward: dL/dtable only; the reference returns
    None for the positions (triplane.py:197) and there is no dL/dx kernel, so positions that require grad are
    refused in forward."""

    @staticmethod
    def forward(ctx, positions, table, encoder):
        out = ops.triplane_encode_fwd(positions, table.detach(), encoder._clayout)
        ctx.encoder = encoder
        ctx.save_for_backward(positions, table)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        positions, table = ctx.saved_tensors
        enc = ctx.encoder
        dy = grad_out.float().contiguous()
        if enc.grad_sink is not None:
            # fused-optimizer path: accumulate straight into the trainer's flat gradient buffer
            ops.triplane_encode_bwd(positions, table.detach(), dy, enc._clayout, enc.grad_sink)
            return None, None, None
        # the gradient G of this one backward, returned once (the reference returns params.grad, triplane.py:197)
        grad_table = torch.zeros(table.numel(), device=table.device, dtype=torch.float32)
        ops.triplane_encode_bwd(positions, table.detach(), dy, enc._clayout, grad_table)
        return None, grad_table.view_as(table), None


class TriPlaneEncoder(torch.nn.Module):

    def __init__(self, base_res: int = 16, max_res: int = 2048, levels: int = 16, feature_per_level: int = 2):
        super().__init__()
        lay = make_triplane_layout(levels, base_res, max_res, feature_per_level)
        self._layout = lay
        self._clayout = lay.as_ctypes()
        self.base_res = base_res
        self.max_res = max_res
        self.levels = levels
        self.feature_per_level = feature_per_level
        self.out_dim = lay.out_dim
        self.log_b = lay.log_b
        self.total_param_size = lay.total_param_size
        self.plane_embedding = torch.nn.Parameter(torch.zeros(self.total_param_size, dtype=torch_type),
                                                  requires_grad=True)
        torch.nn.init.uniform_(self.plane_embedding)   # triplane.py:129-136
        print(f'TriPlane Encoder: base_res={base_res} max_res={max_res} levels={levels} '
              f'feat_per_level={feature_per_level} per_level_scale={self.log_b} '
              f'total_param_size={self.total_param_size} ', file=sys.stderr)
        self.grad_sink = None  # optional fp32 [P] buffer the backward accumulates into

    def forward(self, positions):
        if positions.requires_grad:
            raise NotImplementedError("TriPlaneEncoder has no gradient wrt the positions (the reference returns None "
                                      "there); pass positions that do not require grad")
        return _TriplaneEncode.apply(positions.float().contiguous(), self.plane_embedding, self)

    # ---- kernel-level interface (NGP's grid update, the frame renderers and the graph-captured step) --------------
    emb_dtype = torch.float32
    bwd_raises_inf = True   # the table backward raises GradScaler's inf flag itself, in both feature widths

    def kernel_table(self):
        """The tensor the encode kernel reads (its pointer is tracked by FrameRenderer's graph)."""
        return self.plane_embedding.detach()

    def encode_world(self, xyzs_w, aabb):
        """fp32 [N, out_dim] embedding of world positions, aabb = (xyz_min[3], xyz_max-xyz_min[3]) normalised in the
        kernel; no autograd."""
        return ops.triplane_encode_fwd(xyzs_w.float().contiguous(), self.kernel_table(), self._clayout, aabb=aabb)

    def enqueue_encode_dyn(self, lib, xyzs, table, emb, n_max, n_dev, aabb6, stream):
        """Raw launch of the device-counted encode (FrameRenderer's rounds): pointers in, rc out."""
        return lib.ngp_triplane_encode_fwd_dyn(xyzs, table, ctypes.byref(self._clayout), emb, n_max, n_dev, aabb6,
                                               stream)

    def enqueue_encode_bwd_dyn(self, lib, xyzs, table, demb, grad_table, n_max, n_dev, aabb6, found_inf, stream):
        """Raw launch of the device-counted table backward (the graph-captured training step): grad_table += dL/dtable
        of the first min(n_max, *n_dev) rows; found_inf (may be None) is raised on a non-finite contribution."""
        return lib.ngp_triplane_encode_bwd_dyn(xyzs, table, demb, ctypes.byref(self._clayout), grad_table, n_max,
                                               n_dev, aabb6, found_inf, stream)
