"""Time the voxel-grid model (`--model_name svox`, G = 256, degree 2: 470 M fp32 parameters) on one GPU.

  python scripts/bench_voxel_grid.py [--steps 300] [--rays 8192] [--out bench_voxel_grid.json]

Trains the default VoxelGrid on the analytic synthetic scene for --warm module-path steps (so the occupancy grid and
the sample stream are those of a model in training), then reports:
  - step: NGPTrainer.step (march, voxel forward, composite, backward, fused Adam), median of 3 windows of --steps;
  - the forward, density-only and both backward mappings on one marched batch of --rays rays, each launch timed with
    CUDA events after a 256 MB write that evicts the L2 (median of 20);
  - the fused Adam pass alone over the flat buffer (param | grad | m | v), L2 flushed the same way, with the bytes it
    moves and the bandwidth that implies.
The card's name, power limit and SM clocks are read in the same process."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, flush, reps=20):
    """median ms of fn() over reps launches, each after an L2-evicting write (not timed)."""
    ts = []
    for _ in range(reps):
        flush.add_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warm", type=int, default=500)
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_voxel_grid.py measures the GPU; no CUDA device found")
    from datasets.ray_utils import get_rays
    from modules.intersection import ray_aabb_intersection
    from modules.ray_march import raymarching_train
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
    tr = NGPTrainer(m, lr=1e-2, max_steps=args.warm + 4 * args.steps)
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

    for _ in range(args.warm):
        step()
    torch.cuda.synchronize()
    windows = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            step()
        b.record()
        b.synchronize()
        windows.append(a.elapsed_time(b) / args.steps)

    # one marched batch of the trained model
    data = ds[k % len(ds)]
    o, d = get_rays(data['direction'], data['pose'])
    o, d = o.contiguous(), d.contiguous()
    hits = ray_aabb_intersection(o, d, m.scale)
    rays_a, xyzs, dirs, deltas, ts, _ = raymarching_train(o, d, hits, m.density_bitfield, m.cascades, m.scale, 0.0,
                                                         m.grid_size, MAX_SAMPLES)
    xyzs, dirs = xyzs.float().contiguous(), dirs.float().contiguous()
    S = xyzs.shape[0]
    sh, den = m.sh_fields.detach(), m.density_fields.detach()
    sigma, rgb = ops.voxel_fwd(xyzs, dirs, sh, den, m._clayout)
    dsig, drgb = torch.randn_like(sigma), torch.randn_like(rgb)
    gsh, gden = tr.flat_grad.new_zeros(sh.shape), tr.flat_grad.new_zeros(den.shape)
    flush = torch.zeros(64 << 20, device=dev)    # 256 MB > the 50 MB L2
    t_fwd = timed(lambda: ops.voxel_fwd(xyzs, dirs, sh, den, m._clayout), flush)
    t_den = timed(lambda: ops.voxel_fwd(xyzs, None, None, den, m._clayout), flush)
    t_bw = timed(lambda: ops.voxel_bwd(xyzs, dirs, sigma, rgb, dsig, drgb, m._clayout, gsh, gden,
                                       mapping=ops.VOXEL_BWD_WARP), flush)
    t_bt = timed(lambda: ops.voxel_bwd(xyzs, dirs, sigma, rgb, dsig, drgb, m._clayout, gsh, gden,
                                       mapping=ops.VOXEL_BWD_THREAD), flush)
    del gsh, gden
    tr.found_inf.zero_()
    t_adam = timed(lambda: tr.enqueue_update(), flush, reps=10)
    P = tr.flat_param.numel()
    # the finite check reads the gradient; Adam reads param, grad, m, v and writes param, m, v and the zeroed gradient
    adam_bytes = P * 4 * 9
    res = {
        "card": card(), "G": m.field_size, "sh_degree": m.sh_degree, "params": P, "rays": args.rays,
        "samples_in_batch": S, "warm_steps": args.warm,
        "step_ms_windows": [round(w, 3) for w in windows], "step_ms": round(sorted(windows)[1], 3),
        "fwd_ms": round(t_fwd, 4), "density_only_ms": round(t_den, 4),
        "bwd_warp_per_sample_ms": round(t_bw, 4), "bwd_thread_per_sample_ms": round(t_bt, 4),
        "adam_update_ms": round(t_adam, 3), "adam_bytes": adam_bytes,
        "adam_GBps": round(adam_bytes / (t_adam * 1e-3) / 1e9, 1),
    }
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
