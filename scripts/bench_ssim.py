"""Time SSIM (`ngp_ssim` through `ops.ssim`, DESIGN.md §6e) on one GPU against a torch restatement of torchmetrics'
op sequence (the reference's StructuralSimilarityIndexMeasure(data_range=1)).

  python scripts/bench_ssim.py [--reps 20] [--out bench_ssim.json]

Per shape (800 x 800 with B = 1 and B = 8, 400 x 400 with B = 1; uniform images, target correlated with pred):
  - each call timed with CUDA events after a 256 MB write that evicts the L2 (median of --reps);
  - the bytes the algorithm needs, both images read once (2 x 12 B per pixel), and the bandwidth that implies;
  - the torch restatement (rearrange to [B, 3, H, W], reflect pad by 5, one grouped 11 x 11 conv2d over the five
    stacked moment maps, the formula, crop by 5, mean per image; fp32 convolutions, TF32 off) timed the same way, and
    the largest difference between the two results.
The card's name, power limit and SM clocks are read in the same process."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SHAPES = [(800, 800, 1), (800, 800, 8), (400, 400, 1)]


def torch_ssim(pred, target, H, W):
    """torchmetrics' SSIM (Gaussian window, sigma 1.5, 11 taps, data_range 1) as torch ops, per image."""
    B = pred.shape[0]
    x = pred.reshape(B, H, W, 3).permute(0, 3, 1, 2)
    y = target.reshape(B, H, W, 3).permute(0, 3, 1, 2)
    d = torch.arange(11, device=pred.device, dtype=torch.float32) - 5
    g = torch.exp(-0.5 * (d / 1.5) ** 2)
    g = g / g.sum()
    k = (g[:, None] * g[None, :]).expand(3, 1, 11, 11)
    x, y = F.pad(x, (5, 5, 5, 5), mode="reflect"), F.pad(y, (5, 5, 5, 5), mode="reflect")
    m = F.conv2d(torch.cat((x, y, x * x, y * y, x * y)), k, groups=3).split(B)
    mx, my = m[0], m[1]
    vx, vy, cxy = m[2] - mx * mx, m[3] - my * my, m[4] - mx * my
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    s = (2 * mx * my + c1) * (2 * cxy + c2) / ((mx * mx + my * my + c1) * (vx + vy + c2))
    return s[..., 5:-5, 5:-5].reshape(B, -1).mean(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim.py measures the GPU; no CUDA device found")
    from bench_voxel_grid import card, timed
    from taichi_nerfs_b200 import ops

    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    flush = torch.zeros(64 << 20, device=dev)    # 256 MB > the 50 MB L2
    rows = []
    for H, W, B in SHAPES:
        gen = torch.Generator(device=dev).manual_seed(H + B)
        pred = torch.rand(B, H * W, 3, device=dev, generator=gen)
        target = 0.6 * pred + 0.4 * torch.rand(B, H * W, 3, device=dev, generator=gen)
        ours, ref = ops.ssim(pred, target, H, W), torch_ssim(pred, target, H, W)   # warm-up + agreement
        t_k = timed(lambda: ops.ssim(pred, target, H, W), flush, reps=args.reps)
        t_t = timed(lambda: torch_ssim(pred, target, H, W), flush, reps=args.reps)
        by = B * H * W * 24
        rows.append({"H": H, "W": W, "B": B, "kernel_ms": round(t_k, 4), "bytes": by,
                     "kernel_GBps": round(by / (t_k * 1e-3) / 1e9, 1), "torch_ms": round(t_t, 4),
                     "speedup": round(t_t / t_k, 2), "max_abs_diff": float((ours - ref).abs().max())})
    res = {"card": card(), "reps": args.reps, "shapes": rows}
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
