"""Isolated timing of the fused MLP kernels (CUDA events, L2 flushed between repeats): forward with / without the
save buffer, backward restarting from the saved activations vs recomputing everything."""
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from taichi_nerfs_b200 import ops

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2_190_000
dev = "cuda"
g = torch.Generator(device=dev).manual_seed(0)
emb = torch.randn(n, 32, device=dev, generator=g).half()
dirs = torch.randn(n, 3, device=dev, generator=g)
ws = [torch.randn(s, device=dev, generator=g) * 0.2 for s in ((64, 32), (16, 64), (64, 32), (64, 64), (3, 64))]
dsig = torch.randn(n, device=dev, generator=g) * 1e-2
drgb = (torch.randn(n, 3, device=dev, generator=g) * 1e-2).half()
flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)
_, _, save = ops.mlp_fwd(emb, dirs, ws, with_save=True)


def t(fn, reps=7):
    out = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


for name, fn in [("fwd", lambda: ops.mlp_fwd(emb, dirs, ws)), ("fwd+save", lambda: ops.mlp_fwd(emb, dirs, ws, with_save=True))]:
    fn()
    us = t(fn) * 1e3
    print(f"{name:22s} {us:8.1f} us   (n = {n}; {18816 * n / us / 1e6:6.1f} TFLOP/s, "
          f"{(86 + (40 if 'save' in name else 0)) * n / us / 1e3:6.0f} GB/s algorithmic)", flush=True)
for name, fn in [("bwd recompute", lambda: ops.mlp_bwd(emb, dirs, ws, dsig, drgb)),
                 ("bwd saved", lambda: ops.mlp_bwd(emb, dirs, ws, dsig, drgb, save=save))]:
    fn()
    us = t(fn) * 1e3
    print(f"{name:34s} {us:8.1f} us   (n = {n}; {37632 * n / us / 1e6:6.1f} TFLOP/s)", flush=True)
