"""fp16 multiresolution hash-grid encoder (``--half_opt``) — mirrors
modules/hash_encoder_half.py of the reference (HashEncoder :218-368): fp32 master table of shape
[entries, F], gathers from an fp16 copy with fp16 accumulation, fp32 gradient accumulation.  Everything else is the
fp32 encoder's (modules/hash_encoder.py)."""
from __future__ import annotations

import torch

from . import hash_encoder

torch_type = torch.float16


class HashEncoder(hash_encoder.HashEncoder):

    def _init_table(self, lay):
        # fp32 master [entries, F], U(-1e-4, 1e-4) (hash_encoder_half.py:291-299)
        table = (torch.rand(lay.total_entries, lay.feat_dim, dtype=torch.float32) * 2.0 - 1.0) * 1e-4
        self.hash_table = torch.nn.Parameter(table, requires_grad=True)
        self.register_buffer('hash_grad', torch.zeros_like(table, dtype=torch.float32))
        # fp16 shadow of the master: refreshed lazily (or written directly by the fused Adam pass)
        self._shadow = None
        self._shadow_version = -1

    def _zeroed_table_grad(self):
        # the reference zeroes its persistent `hash_grad` buffer and accumulates into it
        # (hash_encoder_half.py:350-361)
        return self.hash_grad.zero_()

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

    # ---- kernel-level interface: the fp16 copy and fp16 embeddings -----------------------------------------------
    emb_dtype = torch.float16

    def kernel_table(self):
        """The tensor the encode kernel reads (its pointer is tracked by FrameRenderer's graph)."""
        return self.table_f16()
