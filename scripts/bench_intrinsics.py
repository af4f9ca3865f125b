"""What camera intrinsics refinement (--intrinsics_lr, DESIGN.md §6l) costs:

  1. the step: ms/step of the graph-captured step (bench.py's lego_half shapes and init, batch 8192, host-fed batches of
     the analytic scene) with the feature off and on, timed alternately (--runs runs of --steps steps, CUDA events);
     the off arm gets the rays, the on arm their pixels and image indices and forms the rays itself (a pinhole camera of
     the dataset's K at zero correction gives get_ray_directions' table bit for bit).  The on arm trains its
     corrections at learning rate 0, so both arms fit the same field and march the same samples, and the difference is
     the five new nodes (which do the same arithmetic at any correction);
  2. each new kernel alone on the buffers of one real step of the on arm (unproject, pose apply, input gradient,
     intrinsics gradient, Adam), CUDA events, L2 flushed before every launch, median of --reps.

    python scripts/bench_intrinsics.py [--steps 200] [--runs 3] [--reps 21]

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


def build(ds, with_intrinsics):
    import torch
    from modules.networks import NGP
    from taichi_nerfs_b200.intrinsics import Camera, IntrinsicsRefinement
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
    x = None
    if with_intrinsics:
        K = ds.K.double().cpu()
        cam = Camera('PINHOLE', float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
        x = IntrinsicsRefinement(cam, *ds.img_wh, 0.0, ds.poses)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=20000, intrinsics=x)
    fast = StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"], exp_step_factor=cfg["esf"])
    return fast, model


def run(fast, model, batches, first, k):
    import torch
    samples = torch.zeros((), device=fast.dev, dtype=torch.float64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(first, first + k):
        if i % bench.UPDATE_INTERVAL == 0:
            with torch.autocast("cuda", dtype=torch.float16):
                model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
        b = batches[i % len(batches)]
        if fast.intr is not None:
            fast.step(None, None, b["rgb"], img_idxs=b["img_idxs"], pix_idxs=b["pix_idxs"])
        else:
            fast.step(b["rays_o"], b["rays_d"], b["rgb"])
        samples += fast.counter[0].clamp(max=fast.cap)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / k, float(samples) / k


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batches", type=int, default=32)
    ap.add_argument("--warm", type=int, default=64)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=21)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_intrinsics.py measures the H100 path and needs a CUDA device")
    from datasets.ray_utils import get_rays
    from datasets.synthetic import SyntheticLego
    dev = torch.device("cuda", 0)
    gpu = card()
    cfg = bench.CONFIGS["lego_half"]
    ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                       radius=cfg["radius"], scene="analytic").to(dev)
    batches = []
    for i in range(args.batches):
        b = ds[i]
        img = torch.as_tensor(b["img_idxs"], device=dev)
        pix = torch.as_tensor(b["pix_idxs"], device=dev)
        batches.append({"rgb": b["rgb"], "img_idxs": img, "pix_idxs": pix,
                        **dict(zip(("rays_o", "rays_d"), get_rays(b["direction"], b["pose"])))})
    arms = {"off": build(ds, False), "on": build(ds, True)}
    for fast, model in arms.values():
        run(fast, model, batches, 0, args.warm)
    step = {k: [] for k in arms}
    samples = {k: [] for k in arms}
    pos = args.warm
    for _ in range(args.runs):
        for key, (fast, model) in arms.items():
            ms, sm = run(fast, model, batches, pos, args.steps)
            step[key].append(ms)
            samples[key].append(sm)
            pos += args.steps
    fon = arms["on"][0]
    torch.cuda.synchronize()
    S = min(int(fon.counter[0]), fon.cap)
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    kern = {"unproject": time_kernel(fon._k_unproject, flush, args.reps),
            "pose_apply": time_kernel(fon._k_pose_apply_intr, flush, args.reps),
            "input_grad": time_kernel(fon._k_hash_dx, flush, args.reps),
            "intrinsics_grad": time_kernel(fon._k_intr_grad, flush, args.reps),
            "adam": time_kernel(lambda: fon.intr.enqueue_adam(fon.tr), flush, args.reps),
            "head": time_kernel(fon._k_head, flush, args.reps)}
    res = dict(config="lego_half", scene="analytic", card=gpu, batch=bench.BATCH, n_img=fon.intr.n_img, samples=S,
               kernels_per_replay={k: f.kernels_per_replay for k, (f, _) in arms.items()},
               step_ms={k: [round(v, 4) for v in vs] for k, vs in step.items()},
               step_ms_median={k: round(statistics.median(v), 4) for k, v in step.items()},
               samples_per_step={k: [round(v) for v in vs] for k, vs in samples.items()},
               kernel_ms={k: round(v, 4) for k, v in kern.items()})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
