"""What the distortion loss costs in the graph-captured training step (StaticTrainStep(distortion_loss_w=w)), measured on
bench.py's workload shapes (lego_half, garden16: batch 8192, device-sampled batches, overlap mode):

  1. the step: ms/step with w = 0 and w = --w: two captured steps on ONE trainer (so both arms train the same model
     and march comparable sample counts), timed alternately (--runs runs of --steps steps each, CUDA events around the
     replays, the pending update flushed at every switch), with the samples per step of each arm;
  2. the per-ray head alone, on the buffers of one real step: ngp_ray_head_fused (w = 0) and
     ngp_ray_head_fused_distortion (w), CUDA events, L2 flushed before every launch, median of --reps;
  3. the module path (NGPTrainer.step, autograd) with and without extra_loss = w * distortion_loss(res).mean(), on
     batches the graph step drew: the cost of the distortion loss before it was fused.

    python scripts/bench_distortion.py [--configs lego_half garden16] [--w 1e-2] [--steps 200] [--runs 3]

Prints one JSON line per configuration, with the card's name and power limit read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "nvidia-smi unavailable"


def build(cfg_name, ws_d, ds, warm):
    """Graph steps of bench.py's init and shape, one per distortion weight in ws_d, all on one trainer, after `warm`
    steps of the first (density grid updates every bench.UPDATE_INTERVAL steps, as bench.py)."""
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    dev = torch.device("cuda", 0)
    cfg = bench.CONFIGS[cfg_name]
    torch.manual_seed(bench.SEED)
    _, table, ws = bench.init_weights_numpy(bench.SEED, cfg["max_res"], cfg["half"])
    model = NGP(scale=cfg["scale"], max_res=cfg["max_res"], half_opt=cfg["half"]).to(dev)
    with torch.no_grad():
        model.pos_encoder.hash_table.copy_(torch.from_numpy(table).view_as(model.pos_encoder.hash_table))
        for p, wt in zip(bench.mlp_params(model), ws):
            p.copy_(torch.from_numpy(wt))
    model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=20000)
    steps = []
    for w in ws_d:
        fast = StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"], exp_step_factor=cfg["esf"],
                               overlap_optimizer=True, distortion_loss_w=w)
        fast.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=bench.SEED)
        steps.append(fast)
    for i in range(warm):
        _steps(steps[0], model, i, 1)
    steps[0].flush()
    torch.cuda.synchronize()
    return steps, model, trainer


def _steps(fast, model, first, k):
    import torch
    for i in range(first, first + k):
        if i % bench.UPDATE_INTERVAL == 0:
            with torch.autocast("cuda", dtype=torch.float16):
                fast.flush()
                model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
        loss = fast.step_sampled()
    return loss


def time_steps(fast, model, first, k):
    """(ms per step, mean samples per step) of k steps."""
    import torch
    samples = torch.zeros((), device=fast.dev, dtype=torch.float64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(first, first + k):
        _steps(fast, model, i, 1)
        samples += fast.counter[0].clamp(max=fast.cap)
    fast.flush()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k, float(samples) / k


def time_kernel(fn, flush, reps):
    import torch
    out = []
    for _ in range(reps):
        flush.fill_(1)                      # evict L2 (50 MB) before every launch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return statistics.median(out)


def module_path(fast, model, trainer, cfg, w, n_batches, k, runs):
    """ms/step of NGPTrainer.step on n_batches batches the graph step drew (cycled k times), with and without the
    distortion loss, alternated (`runs` times each; the median is reported)."""
    import torch
    from modules.distortion import distortion_loss
    batches = []
    for _ in range(n_batches):
        fast.step_sampled()
        batches.append((fast.rays_o.clone(), fast.rays_d.clone(), fast.gt.clone()))
    fast.flush()
    extra = lambda res: w * distortion_loss(res).mean()  # noqa: E731
    out = {"w0": [], "w": []}
    for _ in range(runs):
        for key, el in (("w0", None), ("w", extra)):
            for b in batches:                               # warm-up of this arm
                trainer.step(*b, cfg["esf"], extra_loss=el)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for i in range(k):
                trainer.step(*batches[i % n_batches], cfg["esf"], extra_loss=el)
            e1.record()
            torch.cuda.synchronize()
            out[key].append(e0.elapsed_time(e1) / k)
    return {key: round(statistics.median(v), 4) for key, v in out.items()}, {key: [round(x, 4) for x in v] for key, v in out.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", nargs="+", default=["lego_half", "garden16"], choices=["lego_half", "garden16"])
    ap.add_argument("--w", type=float, default=1e-2)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--module-steps", type=int, default=100)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_distortion.py measures the H100 path and needs a CUDA device")
    from datasets.synthetic import SyntheticLego
    dev = torch.device("cuda", 0)
    gpu = card()
    for name in args.configs:
        cfg = bench.CONFIGS[name]
        ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                           radius=cfg["radius"]).to(dev)
        ds.build_image_bank()
        (f0, fw), model, trainer = build(name, (0.0, args.w), ds, args.warm)
        arms = {"w0": f0, "w": fw}
        step = {"w0": [], "w": []}
        samples = {"w0": [], "w": []}
        pos = args.warm
        for _ in range(args.runs):                  # alternate the two steps (the counter is only read at the end)
            for key, fast in arms.items():
                ms, sm = time_steps(fast, model, pos, args.steps)
                step[key].append(ms)
                samples[key].append(sm)
                pos += args.steps
        # the head alone on the buffers of one real step of the w arm, both entries
        fast = fw
        fast.step_sampled()
        fast.flush()
        torch.cuda.synchronize()
        S = min(int(fast.counter[0]), fast.cap)      # rows the head reads: the march drops what exceeds the capacity
        truncated = int(fast.counter[1])
        flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
        head = {}
        for key, wv in (("w0", 0.0), ("w", args.w), ("w0_again", 0.0), ("w_again", args.w)):
            fast.distortion_w = wv
            head[key] = time_kernel(fast._k_head, flush, args.reps)
        fast.distortion_w = args.w
        del flush
        mod, mod_runs = module_path(fast, model, trainer, cfg, args.w, 4, args.module_steps, args.runs)
        res = dict(config=name, card=gpu, w=args.w, batch=bench.BATCH, head_samples=S, head_capacity=fast.cap, head_rays_truncated=truncated,
                   step_ms={k: [round(v, 4) for v in vs] for k, vs in step.items()},
                   step_ms_median={k: round(statistics.median(v), 4) for k, v in step.items()},
                   samples_per_step={k: [round(v) for v in vs] for k, vs in samples.items()},
                   head_ms={k: round(v, 4) for k, v in head.items()},
                   module_step_ms=mod, module_step_ms_runs=mod_runs)
        print(json.dumps(res), flush=True)
        del arms, fast, f0, fw, model, trainer
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
