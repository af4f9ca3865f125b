"""What error-map ray sampling (--ray_sampling_strategy error_map, DESIGN.md §6j) costs and what it gives:

  1. the step: ms/step of the graph-captured step (bench.py's lego_half shapes and init, batch 8192, host-fed batches of
     the analytic scene) with the feature off and on, timed alternately (--runs runs of --steps steps, CUDA events);
     the on arm's batches are drawn from a uniform map and gathered beforehand, so the difference is the two new nodes;
  2. each new kernel alone on the buffers of one real step of the on arm (sampler, accumulate, gradient weight) and the
     rebuild of a 100-image map, CUDA events, L2 flushed before every launch, median of --reps;
  3. held-out PSNR against the teacher Lego (taichi_nerfs_b200.psnr.train_vs_teacher, graph step) after 1000, 2000 and
     3000 steps for both strategies and every --seeds (one training per step count: the cosine schedule ends at it).

    python scripts/bench_error_map.py [--steps 200] [--runs 3] [--seeds 23 24 25] [--no-psnr]

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


def build(ds, em):
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
    fast = StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"], exp_step_factor=cfg["esf"],
                           error_map=em)
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
        if fast.em is not None:
            fast.step(b["rays_o"], b["rays_d"], b["rgb"], ray_w=b["w"], img_idxs=b["img_idxs"],
                      pix_idxs=b["pix_idxs"])
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
    ap.add_argument("--seeds", type=int, nargs="+", default=[23, 24, 25])
    ap.add_argument("--no-psnr", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_error_map.py measures the H100 path and needs a CUDA device")
    from datasets.ray_utils import get_rays
    from datasets.synthetic import SyntheticLego
    from taichi_nerfs_b200.error_map import ErrorMap
    dev = torch.device("cuda", 0)
    gpu = card()
    cfg = bench.CONFIGS["lego_half"]
    ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                       radius=cfg["radius"], scene="analytic").to(dev)
    em = ErrorMap(len(ds.poses), *ds.img_wh, seed=bench.SEED, device=dev)
    batches = {"off": [], "on": []}
    for i in range(args.batches):
        b = ds[i]
        batches["off"].append({"rgb": b["rgb"], **dict(zip(("rays_o", "rays_d"), get_rays(b["direction"], b["pose"])))})
        img, pix, w = em.draw(bench.BATCH, i)
        g = ds.gather(img, pix)
        batches["on"].append({"rgb": g["rgb"], "w": w, "img_idxs": img, "pix_idxs": pix,
                              **dict(zip(("rays_o", "rays_d"), get_rays(g["direction"], g["pose"])))})
    arms = {"off": build(ds, None), "on": build(ds, em)}
    for key, (fast, model) in arms.items():
        run(fast, model, batches[key], 0, args.warm)
    step = {k: [] for k in arms}
    samples = {k: [] for k in arms}
    pos = args.warm
    for _ in range(args.runs):
        for key, (fast, model) in arms.items():
            ms, sm = run(fast, model, batches[key], pos, args.steps)
            step[key].append(ms)
            samples[key].append(sm)
            pos += args.steps
    fon = arms["on"][0]
    torch.cuda.synchronize()
    S = min(int(fon.counter[0]), fon.cap)
    flush = torch.empty(256 * 1024 * 1024, device=dev, dtype=torch.uint8)
    out = (fon.em_img.clone(), fon.em_pix.clone(), fon.ray_w.clone())
    kern = {"sample": time_kernel(lambda: em.draw(bench.BATCH, 7, out=out), flush, args.reps),
            "accumulate": time_kernel(fon._k_em_accumulate, flush, args.reps),
            "grad_weight": time_kernel(fon._k_grad_weight, flush, args.reps),
            "rebuild": time_kernel(em.rebuild, flush, args.reps),
            "head": time_kernel(fon._k_head, flush, args.reps)}
    res = dict(config="lego_half", scene="analytic", card=gpu, batch=bench.BATCH, n_img=em.n_img, tiles=em.T,
               samples=S, step_ms={k: [round(v, 4) for v in vs] for k, vs in step.items()},
               step_ms_median={k: round(statistics.median(v), 4) for k, v in step.items()},
               samples_per_step={k: [round(v) for v in vs] for k, vs in samples.items()},
               kernel_ms={k: round(v, 4) for k, v in kern.items()})
    if not args.no_psnr:
        from datasets.teacher import load_teacher
        from taichi_nerfs_b200.psnr import train_vs_teacher
        teacher = load_teacher(dev)
        if teacher is None:
            raise SystemExit("teacher model not staged: run __graft_entry__.build()")
        psnr = {}
        for strategy in ("all_images", "error_map"):
            for steps in (1000, 2000, 3000):
                psnr[f"{strategy}@{steps}"] = [round(train_vs_teacher(dev, steps=steps, seed=s, teacher=teacher,
                                                                      ray_sampling=strategy)["psnr"], 3)
                                               for s in args.seeds]
        res["psnr"] = psnr
        res["seeds"] = args.seeds
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
