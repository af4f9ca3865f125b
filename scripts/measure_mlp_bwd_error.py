"""Measured error of the fused MLP backward against the oracle (per gradient block), to set the test tolerances."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O  # noqa: E402
from taichi_nerfs_b200 import ops  # noqa: E402

T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
for n in (5000, 40000):
    for saved in (False, True):
        rng = np.random.default_rng(35)
        emb = (rng.standard_normal((n, 32)) * 0.5).astype(np.float16)
        dirs = rng.standard_normal((n, 3)).astype(np.float32)
        shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
        ws = [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]
        dsig = (rng.standard_normal(n) * 0.1).astype(np.float32)
        drgb = (rng.standard_normal((n, 3)) * 0.1).astype(np.float16)
        demb_ref, gw_ref = O.mlp_bwd(emb, dirs, ws, dsig, drgb)
        save = None
        if saved:
            _, _, save = ops.mlp_fwd(T(emb), T(dirs), [T(w) for w in ws], with_save=True)
        demb, gw = ops.mlp_bwd(T(emb), T(dirs), [T(w) for w in ws], T(dsig), T(drgb), save=save)
        demb, gw = demb.float().cpu().numpy(), gw.cpu().numpy()
        demb_ref = demb_ref.astype(np.float32)
        offs = np.cumsum([0, 2048, 1024, 2048, 4096, 192])
        blocks = [np.abs(gw[a:b] - gw_ref[a:b]).max() / np.abs(gw_ref[a:b]).max() for a, b in zip(offs[:-1], offs[1:])]
        print(f"n={n} saved={saved}: demb max err / max = {np.abs(demb - demb_ref).max() / np.abs(demb_ref).max():.2e}, "
              f"99.9th pct {np.percentile(np.abs(demb - demb_ref), 99.9) / np.abs(demb_ref).max():.2e}; dW blocks (max err / block max): "
              + ", ".join(f"{b:.2e}" for b in blocks))
