"""What --random_bg costs in the graph-captured training step (StaticTrainStep(random_bg=True), DESIGN.md §6f), on
bench.py's lego_half shape (batch 8192, overlap mode):

  1. the step: ms/step with random_bg off and on, two captured steps on ONE trainer (both arms train the same model
     and march comparable sample counts), fed the same host batches (step(rays_o, rays_d, rgb, alpha): the device
     sampler does not take random_bg), timed alternately (--runs runs of --steps steps each, CUDA events around the
     steps, the pending update flushed at every switch), median and spread;
  2. the per-ray head alone on the buffers of one real step: the constant-background head, and the colour draw plus
     the random-background head, CUDA events, L2 flushed before every launch, median of --reps.

    python scripts/bench_random_bg.py [--steps 200] [--runs 3]

Prints one JSON line with the card's name, power limit and max SM clock read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import bench  # noqa: E402
from bench_distortion import card, time_kernel  # noqa: E402


def build(ds, warm, batches):
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
    arms = {key: StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"],
                                 exp_step_factor=cfg["esf"], overlap_optimizer=True, random_bg=on, bg_seed=bench.SEED)
            for key, on in (("off", False), ("on", True))}
    run(arms["off"], model, batches, 0, warm)
    arms["off"].flush()
    torch.cuda.synchronize()
    return arms, model


def run(fast, model, batches, first, k):
    import torch
    for i in range(first, first + k):
        if i % bench.UPDATE_INTERVAL == 0:
            with torch.autocast("cuda", dtype=torch.float16):
                fast.flush()
                model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
        o, d, rgb, a = batches[i % len(batches)]
        fast.step(o, d, rgb, alpha=a if fast.random_bg else None)


def time_steps(fast, model, batches, first, k):
    import torch
    samples = torch.zeros((), device=fast.dev, dtype=torch.float64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(first, first + k):
        run(fast, model, batches, i, 1)
        samples += fast.counter[0].clamp(max=fast.cap)
    fast.flush()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k, float(samples) / k


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--batches", type=int, default=16)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_random_bg.py measures the H100 path and needs a CUDA device")
    from datasets.ray_utils import get_rays
    from datasets.synthetic import SyntheticLego
    dev = torch.device("cuda", 0)
    cfg = bench.CONFIGS["lego_half"]
    ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                       radius=cfg["radius"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(bench.SEED)
    batches = []
    for i in range(args.batches):
        b = ds[i]
        o, d = get_rays(b["direction"], b["pose"])
        batches.append((o.contiguous(), d.contiguous(), b["rgb"],
                        torch.rand(bench.BATCH, device=dev, generator=g)))
    arms, model = build(ds, args.warm, batches)
    step = {"off": [], "on": []}
    samples = {"off": [], "on": []}
    pos = args.warm
    for _ in range(args.runs):
        for key, fast in arms.items():
            ms, sm = time_steps(fast, model, batches, pos, args.steps)
            step[key].append(ms)
            samples[key].append(sm)
            pos += args.steps
    fast = arms["on"]
    run(fast, model, batches, pos, 1)
    fast.flush()
    torch.cuda.synchronize()
    S = min(int(fast.counter[0]), fast.cap)
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    head = {}
    for key, on in (("off", False), ("on", True), ("off_again", False), ("on_again", True)):
        fast.random_bg = on        # same buffers; "on" launches the colour draw and the random-background head
        head[key] = time_kernel(fast._k_head, flush, args.reps)
    fast.random_bg = True
    res = dict(config="lego_half", card=card(), batch=bench.BATCH, head_samples=S,
               step_ms={k: [round(v, 4) for v in vs] for k, vs in step.items()},
               step_ms_median={k: round(statistics.median(v), 4) for k, v in step.items()},
               step_ms_spread={k: round(max(v) - min(v), 4) for k, v in step.items()},
               samples_per_step={k: [round(v) for v in vs] for k, vs in samples.items()},
               head_ms={k: round(v, 4) for k, v in head.items()})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
