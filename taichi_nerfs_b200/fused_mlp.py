"""Autograd front end of the fused wgmma NGP MLP (csrc/mlp.cu).

Used by ``modules.networks.NGP.forward`` whenever the stock architecture is configured (32-d
embedding, 64-wide sigma net with 16 outputs, 2x64 rgb net): one kernel launch replaces the five
nn.Linear calls + SH encoder + activations of the reference (modules/networks.py:136-166), and one
launch replaces their autograd graph.  Parameters stay the nn.Linear weights of the model (same
state_dict keys); gradients flow back to them through torch.autograd as usual.
"""
from __future__ import annotations

import torch

from . import _lib, ops

_SPLITS = (64 * 32, 16 * 64, 64 * 32, 64 * 64, 3 * 64)
_SHAPES = ((64, 32), (16, 64), (64, 32), (64, 64), (3, 64))


def available() -> bool:
    try:
        _lib.load()
        return True
    except (OSError, _lib.NgpError):
        return False


class _FusedMLP(torch.autograd.Function):

    @staticmethod
    def forward(ctx, emb, dirs, w1, w2, w3, w4, w5):
        emb = emb.contiguous()
        dirs = dirs.float().contiguous()
        ws = [w.detach().float().contiguous() for w in (w1, w2, w3, w4, w5)]
        need_bwd = any(ctx.needs_input_grad)
        if need_bwd:   # keep h + the fp16 sigmoid output (40 B/sample): the backward then skips two serial layers
            sigmas, rgbs, save = ops.mlp_fwd(emb, dirs, ws, with_save=True)
            ctx.save_for_backward(emb, dirs, save, *ws)
        else:
            sigmas, rgbs = ops.mlp_fwd(emb, dirs, ws)
        return sigmas, rgbs

    @staticmethod
    def backward(ctx, d_sigmas, d_rgbs):
        emb, dirs, save, *ws = ctx.saved_tensors
        n = emb.shape[0]
        if d_sigmas is None:
            d_sigmas = torch.zeros(n, device=emb.device, dtype=torch.float32)
        if d_rgbs is None:
            d_rgbs = torch.zeros(n, 3, device=emb.device, dtype=torch.float16)
        demb, gw = ops.mlp_bwd(emb, dirs, ws, d_sigmas, d_rgbs, save=save)
        grads = [g.view(s) for g, s in zip(torch.split(gw, _SPLITS), _SHAPES)]
        return (demb if ctx.needs_input_grad[0] else None, None, *grads)


def mlp_weights(model):
    return (model.xyz_encoder.hidden_layers[0].weight, model.xyz_encoder.output_layer.weight,
            model.rgb_net.hidden_layers[0].weight, model.rgb_net.hidden_layers[1].weight,
            model.rgb_net.output_layer.weight)


def ngp_mlp_forward(model, embedding, dirs):
    """(embedding [N,32], un-normalised dirs [N,3]) -> (sigmas [N] fp32, rgbs [N,3] fp16)."""
    return _FusedMLP.apply(embedding, dirs, *mlp_weights(model))


@torch.no_grad()
def ngp_density(model, embedding):
    """sigma only (occupancy-grid updates): runs the fused kernel with a dummy direction."""
    dirs = torch.zeros(embedding.shape[0], 3, device=embedding.device, dtype=torch.float32)
    dirs[:, 2] = 1.0
    sigmas, _ = ops.mlp_fwd(embedding.contiguous(), dirs, [w.detach() for w in mlp_weights(model)])
    return sigmas
