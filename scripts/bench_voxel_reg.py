"""Time the voxel-grid regularisers (`ngp_voxel_reg`: total variation + sparsity, DESIGN.md §6d) on one GPU, at the
default VoxelGrid (G = 256, degree 2) on the analytic scene.

  python scripts/bench_voxel_reg.py [--steps 200] [--warm 500] [--weights 0.01 0.01 0.01] [--out bench_voxel_reg.json]

Trains --warm module-path steps without the regularisers (so the occupancy grid and the fields are those of a model
in training), then reports:
  - the kernel alone over B (all three terms on, and TV_sh alone), each launch timed with CUDA events after a 256 MB
    write that evicts the L2 (median of 20);
  - the bytes the kernel has to move, 4 |B| C (read the field) + 8 |B| C (read and write the gradient), C = 3D + 1
    channels, and the bandwidth that implies;
  - NGPTrainer.step with and without the regularisers, alternated in this process: 3 windows of --steps each.
The card's name, power limit and SM clocks are read in the same process."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warm", type=int, default=500)
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--weights", type=float, nargs=3, default=[0.01, 0.01, 0.01])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_voxel_reg.py measures the GPU; no CUDA device found")
    from bench_voxel_grid import card, timed
    from datasets.ray_utils import get_rays
    from modules.rendering import MAX_SAMPLES
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200 import ops
    from taichi_nerfs_b200.trainer import NGPTrainer
    from test_gpu_e2e import _small_dataset

    dev = torch.device("cuda")
    torch.manual_seed(23)
    ds = _small_dataset(root_dir='', split='train', downsample=1.0, seed=23).to(dev)
    ds.batch_size = args.rays
    ds.ray_sampling_strategy = 'all_images'
    m = VoxelGrid().to(dev)
    m.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    weights = tuple(args.weights)
    tr = NGPTrainer(m, lr=1e-2, max_steps=args.warm + 7 * args.steps, voxel_reg=weights)
    thr = 0.01 * MAX_SAMPLES / 3 ** 0.5
    k = 0

    def step():
        nonlocal k
        data = ds[k % len(ds)]
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            if k % 16 == 0:
                m.update_density_grid(thr, warmup=k < 256)
        o, d = get_rays(data['direction'], data['pose'])
        tr.step(o, d, data['rgb'])
        k += 1

    tr.voxel_reg = None                     # warm up without the regularisers
    for _ in range(args.warm):
        step()
    torch.cuda.synchronize()
    windows = {"off": [], "on": []}
    for _ in range(3):
        for mode in ("off", "on"):
            tr.voxel_reg = weights if mode == "on" else None
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                step()
            b.record()
            b.synchronize()
            windows[mode].append(a.elapsed_time(b) / args.steps)

    block = m._reg_block
    nodes = (block[3] - block[0]) * (block[4] - block[1]) * (block[5] - block[2])
    Cn = 3 * m.sh_dim + 1
    sh, den = m.sh_fields.detach(), m.density_fields.detach()
    gsh, gden = torch.zeros_like(sh), torch.zeros_like(den)
    flush = torch.zeros(64 << 20, device=dev)    # 256 MB > the 50 MB L2
    t_all = timed(lambda: ops.voxel_reg(sh, den, m._clayout, block, weights, gsh, gden, loss_scale=1.0), flush)
    t_sh = timed(lambda: ops.voxel_reg(sh, den, m._clayout, block, (0.0, 1.0, 0.0), gsh, gden, loss_scale=1.0), flush)
    by_all = nodes * Cn * 12
    by_sh = nodes * (Cn - 1) * 12
    med = lambda v: round(sorted(v)[1], 3)  # noqa: E731
    res = {
        "card": card(), "G": m.field_size, "sh_degree": m.sh_degree, "block": list(block), "block_nodes": nodes,
        "channels": Cn, "weights": list(weights), "rays": args.rays, "warm_steps": args.warm,
        "kernel_ms": round(t_all, 4), "kernel_bytes": by_all, "kernel_GBps": round(by_all / (t_all * 1e-3) / 1e9, 1),
        "kernel_tv_sh_only_ms": round(t_sh, 4), "kernel_tv_sh_only_GBps": round(by_sh / (t_sh * 1e-3) / 1e9, 1),
        "step_ms_off_windows": [round(w, 3) for w in windows["off"]],
        "step_ms_on_windows": [round(w, 3) for w in windows["on"]],
        "step_ms_off": med(windows["off"]), "step_ms_on": med(windows["on"]),
    }
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
