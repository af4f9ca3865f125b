"""What depth supervision costs in the graph-captured training step (StaticTrainStep(depth_loss_w=w), DESIGN.md §6h),
on bench.py's lego_half shapes (batch 8192, --half_opt hash model, overlap mode):

  1. the step: ms/step with w = 0 and w = --w: two captured steps on ONE trainer, fed the same host batches of the
     analytic scene with their z-depth targets (the device-sampled batches carry no depth), timed alternately (--runs
     runs of --steps steps each, CUDA events around the steps, the pending update flushed at every switch), with the
     samples per step of each arm;
  2. the per-ray head alone, on the buffers of one real step of the w arm: ngp_ray_head_fused (w = 0) and
     ngp_ray_head_fused_depth (w), CUDA events, L2 flushed before every launch, median of --reps.

    python scripts/bench_depth.py [--w 0.1] [--steps 200] [--runs 3]

Prints one JSON line, with the card's name and power limit read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
from bench_distortion import card, time_kernel  # noqa: E402


def build(ws_z, ds):
    """Graph steps of bench.py's lego_half init, one per depth weight in ws_z, all on one trainer."""
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    dev = torch.device("cuda", 0)
    cfg = bench.CONFIGS["lego_half"]
    torch.manual_seed(bench.SEED)
    _, table, ws = bench.init_weights_numpy(bench.SEED, cfg["max_res"], cfg["half"])
    model = NGP(scale=cfg["scale"], max_res=cfg["max_res"], half_opt=cfg["half"]).to(dev)
    with torch.no_grad():
        model.pos_encoder.hash_table.copy_(torch.from_numpy(table).view_as(model.pos_encoder.hash_table))
        for p, wt in zip(bench.mlp_params(model), ws):
            p.copy_(torch.from_numpy(wt))
    model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=20000)
    steps = [StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"], exp_step_factor=cfg["esf"],
                             overlap_optimizer=True, depth_loss_w=w) for w in ws_z]
    return steps, model


def run(fast, model, batches, first, k):
    """(ms per step, mean samples per step) of k steps on the cycled batches."""
    import torch
    from datasets.ray_utils import get_rays
    samples = torch.zeros((), device=fast.dev, dtype=torch.float64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(first, first + k):
        if i % bench.UPDATE_INTERVAL == 0:
            with torch.autocast("cuda", dtype=torch.float16):
                fast.flush()
                model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
        b = batches[i % len(batches)]
        o, d = get_rays(b["direction"], b["pose"])
        fast.step(o, d, b["rgb"], depth=b["depth"] if fast.depth_w > 0 else None)
        samples += fast.counter[0].clamp(max=fast.cap)
    fast.flush()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k, float(samples) / k


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--w", type=float, default=0.1)
    ap.add_argument("--batches", type=int, default=32)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=21)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth.py measures the H100 path and needs a CUDA device")
    from datasets.synthetic import SyntheticLego
    dev = torch.device("cuda", 0)
    gpu = card()
    cfg = bench.CONFIGS["lego_half"]
    ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                       radius=cfg["radius"], scene="analytic", with_depth=True).to(dev)
    batches = [ds[i] for i in range(args.batches)]
    (f0, fw), model = build((0.0, args.w), ds)
    run(fw, model, batches, 0, args.warm)
    arms = {"w0": f0, "w": fw}
    step = {"w0": [], "w": []}
    samples = {"w0": [], "w": []}
    pos = args.warm
    for _ in range(args.runs):
        for key, fast in arms.items():
            ms, sm = run(fast, model, batches, pos, args.steps)
            step[key].append(ms)
            samples[key].append(sm)
            pos += args.steps
    # the head alone on the buffers of one real step of the w arm, both entries
    from datasets.ray_utils import get_rays
    b = batches[0]
    fw.step(*get_rays(b["direction"], b["pose"]), b["rgb"], depth=b["depth"])
    fw.flush()
    torch.cuda.synchronize()
    S = min(int(fw.counter[0]), fw.cap)
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    head = {}
    for key, wv in (("w0", 0.0), ("w", args.w), ("w0_again", 0.0), ("w_again", args.w)):
        fw.depth_w = wv
        head[key] = time_kernel(fw._k_head, flush, args.reps)
    fw.depth_w = args.w
    res = dict(config="lego_half", scene="analytic", card=gpu, w=args.w, batch=bench.BATCH, head_samples=S,
               head_rays_truncated=int(fw.counter[1]),
               step_ms={k: [round(v, 4) for v in vs] for k, vs in step.items()},
               step_ms_median={k: round(statistics.median(v), 4) for k, v in step.items()},
               samples_per_step={k: [round(v) for v in vs] for k, vs in samples.items()},
               head_ms={k: round(v, 4) for k, v in head.items()})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
