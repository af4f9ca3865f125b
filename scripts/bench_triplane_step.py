"""The tri-plane model in the graph-captured training step: step time against the stock hash model and against the
module path, and the five network kernels one by one.

Prints one JSON line:
  gpu       name, power limit and SM clock (nvidia-smi, read in this run; the SM clock again right after the timed steps)
  graph     StaticTrainStep(overlap_optimizer=True).step_sampled(), 8192 rays, bench.py's recipe (random-init model,
            occupancy after one warm-up grid update, training set resident, batch drawn on the device) of the tri-plane
            model (L = 8, F = 4, max_res 1024, fp32) and of the stock --half_opt hash model, alternated round by round:
            ms/step and rays/s per round and their median, rows marched per step, rays truncated or dropped for capacity
  module    the same tri-plane model through NGPTrainer.step on batches of the same training set
  kernels   encode fwd, MLP fwd, ray head, MLP bwd, encode bwd alone on the buffers of a real tri-plane step; CUDA
            events, L2 flushed between repeats, median of --reps

No grid update runs inside the timed windows (bench.py amortises one every 16 steps on top of the step time).  Every
timed shape is warmed up; a window is --steps steps (seconds, not milliseconds).

Usage: python scripts/bench_triplane_step.py [--steps 300] [--rounds 3] [--reps 7]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_triplane import gpu_info  # noqa: E402

BATCH, SEED, CAP = 8192, 23, 384
DENSITY_THRESHOLD = 0.01 * 1024 / 3 ** 0.5


def make_arm(kind, ds, graph=True):
    from modules.networks import NGP
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    torch.manual_seed(SEED)
    if kind == "triplane":
        model = NGP(scale=0.5, max_res=1024, pos_encoder_type="triplane").cuda()
    else:
        model = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    with torch.autocast("cuda", dtype=torch.float16):
        model.update_density_grid(DENSITY_THRESHOLD, warmup=True)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=20000)
    fast = None
    if graph:
        fast = StaticTrainStep(trainer, BATCH, samples_per_ray_capacity=CAP, overlap_optimizer=True)
        fast.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=SEED)
    return model, trainer, fast


def timed_steps(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def bench_graph(ds, steps, rounds):
    arms = {k: make_arm(k, ds) for k in ("triplane", "hash")}
    ms = {k: [] for k in arms}
    for _, _, fast in arms.values():
        for _ in range(20):
            fast.step_sampled()
    for _ in range(rounds):
        for k, (_, _, fast) in arms.items():
            ms[k].append(timed_steps(lambda i: fast.step_sampled(), steps))
    out = {}
    for k, (_, _, fast) in arms.items():
        rows, dropped = (int(v) for v in fast.stats())
        med = float(np.median(ms[k]))
        out[k] = {"ms_per_step_median": med, "ms_per_step": ms[k], "rays_per_s_median": BATCH / med * 1e3,
                  "rows_last_step": rows, "capacity_rows": fast.cap, "rays_truncated_or_dropped": dropped,
                  "kernels_per_replay": fast.kernels_per_replay_sampled, "inf_at_source": fast.inf_at_source}
    return out, arms


def bench_module(ds, steps, rounds):
    from datasets.ray_utils import get_rays
    _, trainer, _ = make_arm("triplane", ds, graph=False)

    def step(i):
        b = ds[i]
        o, d = get_rays(b["direction"], b["pose"])
        trainer.step(o, d, b["rgb"])
    for i in range(10):
        step(i)
    ms = [timed_steps(step, steps) for _ in range(rounds)]
    med = float(np.median(ms))
    return {"ms_per_step_median": med, "ms_per_step": ms, "rays_per_s_median": BATCH / med * 1e3}


def time_kernel(fn, reset=None, reps=7):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > 50 MB of L2
    fn()
    times = []
    for _ in range(reps):
        if reset is not None:
            reset()
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def bench_kernels(fast, reps):
    """The five network kernels on the buffers the last step left (its march, its dsigma / drgb)."""
    fast.flush()
    torch.cuda.synchronize()
    tr = fast.tr
    rows = int(fast.counter[0])
    clear = lambda: (tr.flat_grad.zero_(), tr.found_inf.zero_())   # noqa: E731
    out = {"rows": min(rows, fast.cap), "capacity_rows": fast.cap,
           "encode_fwd_ms": time_kernel(fast._k_hash_fwd, reps=reps),
           "mlp_fwd_ms": time_kernel(fast._k_mlp_fwd, reps=reps),
           "head_ms": time_kernel(fast._k_head, reset=fast.loss_sum.zero_, reps=reps),
           "mlp_bwd_ms": time_kernel(fast._k_mlp_bwd, reset=clear, reps=reps),
           "encode_bwd_ms": time_kernel(fast._k_hash_bwd, reset=clear, reps=reps)}
    clear()
    out["encode_bwd_ns_per_row"] = out["encode_bwd_ms"] * 1e6 / max(out["rows"], 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    if args.rounds < 3 or args.reps < 5:
        raise SystemExit("at least 3 rounds and 5 repeats: a difference is only trusted against the spread")
    if not torch.cuda.is_available():
        raise SystemExit("bench_triplane_step.py needs a CUDA device")
    from datasets.synthetic import SyntheticLego
    from taichi_nerfs_b200 import _lib
    _lib.load()
    result = {"gpu": gpu_info(), "batch": BATCH, "steps_per_window": args.steps}
    ds = SyntheticLego(batch_size=BATCH, seed=SEED, img_wh=(800, 800), focal=1111.111, radius=1.4).to("cuda")
    ds.build_image_bank()
    result["graph"], arms = bench_graph(ds, args.steps, args.rounds)
    result["gpu"]["sm_clock_after_steps"] = gpu_info().get("sm_clock")
    result["kernels"] = bench_kernels(arms["triplane"][2], args.reps)
    result["hash_kernels"] = bench_kernels(arms["hash"][2], args.reps)
    del arms
    torch.cuda.empty_cache()
    result["module"] = bench_module(ds, max(args.steps // 4, 20), args.rounds)
    result["graph_over_module"] = result["module"]["ms_per_step_median"] / \
        result["graph"]["triplane"]["ms_per_step_median"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
