"""Is the hash-grid scatter bounded by how much of its table gradient L2 holds?  Three experiments on the real sample
stream of the graph-captured training step (xyzs[:S], demb[:S] after --steps steps, as scripts/hash_corner_reuse.py
--source gpu reads it), all timed with CUDA events (median of --reps launches), each with L2 flushed before every
launch and without:

  1. footprint A/B: the same xyz / dL/demb through the all-levels backward with the real layout (T = 2^19: 43.6 MiB of
     fp32 gradient at max_res 1024) and with the same layout at T = 2^16 (~8x smaller), and the same A/B for the fp16
     forward gather.  Time per request = time / (requests the kernel issues for that layout, hash_corner_reuse).
  2. per-level and per-level-group backward launches (ngp_hash_encode_bwd_levels) against the all-levels launch;
  3. --config garden16: the same on the garden-shape stream (max_res 4096), all-levels backward timed three times.

    python scripts/hash_l2_probe.py [--config lego_half|garden16] [--steps 25]

Request counts come from a CPU model of the kernels' lane walk (hash_corner_reuse.count_level) on the first
--count-samples samples, scaled to S; the backward's skip of rows whose dL/demb is zero is not modelled.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
import hash_corner_reuse as hcr  # noqa: E402
from taichi_nerfs_b200.layout import make_hash_layout  # noqa: E402

# candidate level groups: the issue's split, then greedy plans at 1/2, 1/3 and 1/4 of a 50 MiB L2 (lego_half layout)
GROUPS = [(0, 6), (6, 9), (9, 12), (12, 14), (14, 16), (0, 11), (11, 16), (0, 9), (12, 15), (15, 16), (0, 8), (8, 10),
          (10, 12)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "nvidia-smi unavailable"


def gpu_stream(cfg_name, steps):
    """(xyz [S, 3] fp32 world positions, demb [S, 32], aabb6) of the graph step after `steps` steps."""
    import torch
    from datasets.synthetic import SyntheticLego
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
        for p, w in zip(bench.mlp_params(model), ws):
            p.copy_(torch.from_numpy(w))
    ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                       radius=cfg["radius"]).to(dev)
    model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=20000)
    fast = StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"], exp_step_factor=cfg["esf"])
    ds.build_image_bank()
    fast.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=bench.SEED)
    for i in range(steps):
        if i % bench.UPDATE_INTERVAL == 0:
            with torch.autocast("cuda", dtype=torch.float16):
                fast.flush()
                model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
        fast.step_sampled()
    fast.flush()
    torch.cuda.synchronize()
    S = int(fast.counter[0])
    return fast.xyzs[:S].clone(), fast.demb[:S].clone(), fast.aabb6


def counts(lay, xn, S):
    """per level: (backward red requests, forward gather loads), scaled from len(xn) samples to S"""
    k = S / xn.shape[0]
    out = []
    for level in range(lay.levels):
        r = hcr.count_level(lay, level, xn)
        out.append((r["bwd_new"] * k, r["old"] * k))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", choices=("lego_half", "garden16"), default="lego_half")
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--count-samples", type=int, default=1 << 21)
    args = ap.parse_args()
    print(f"card: {card()}")
    cfg = bench.CONFIGS[args.config]
    lay19 = make_hash_layout(2 ** 19, 16, 16, cfg["max_res"], 2)
    lay16 = make_hash_layout(2 ** 16, 16, 16, cfg["max_res"], 2)
    mib = lambda lay, b: lay.total_entries * 2 * b / 2 ** 20  # noqa: E731
    print(f"{args.config}: gradient T=2^19 {mib(lay19, 4):.1f} MiB, T=2^16 {mib(lay16, 4):.1f} MiB; "
          f"fp16 table {mib(lay19, 2):.1f} / {mib(lay16, 2):.1f} MiB")

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the probe times kernels on the GPU (the layouts above are all it can show)")
    from taichi_nerfs_b200._lib import F16, check, load
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    print(f"device: {props.name}, {props.multi_processor_count} SMs, L2 {props.L2_cache_size / 2 ** 20:.1f} MiB")

    xyz, demb, aabb6 = gpu_stream(args.config, args.steps)
    S = xyz.shape[0]
    n_cnt = min(S, args.count_samples)
    lo = np.asarray(aabb6[:3], np.float32)
    span = np.asarray(aabb6[3:], np.float32)
    xn = ((xyz[:n_cnt].cpu().numpy() - lo) / span).astype(np.float32)
    c19, c16 = counts(lay19, xn, S), counts(lay16, xn, S)
    print(f"S = {S} samples after {args.steps} steps; request counts from the first {n_cnt} samples, scaled")

    L = load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    clay = {19: lay19.as_ctypes(), 16: lay16.as_ctypes()}
    grad = {k: torch.zeros(lay.total_entries * 2, device=dev) for k, lay in ((19, lay19), (16, lay16))}
    rng = torch.Generator(device=dev).manual_seed(bench.SEED)
    table = {k: ((torch.rand(lay.total_entries * 2, device=dev, generator=rng) * 2 - 1) * 1e-4).half()
             for k, lay in ((19, lay19), (16, lay16))}
    emb = torch.empty(S, 32, device=dev, dtype=torch.float16)
    flush_buf = torch.empty(256 << 20, device=dev, dtype=torch.uint8)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731

    def bwd(T, a=0, b=16):
        return lambda: check(L.ngp_hash_encode_bwd_levels(p(xyz), p(demb), F16, C.byref(clay[T]), p(grad[T]), S, None,
                                                          aabb6, a, b, None, st), "bwd")

    def fwd(T):
        return lambda: check(L.ngp_hash_encode_fwd_dyn(p(xyz), p(table[T]), C.byref(clay[T]), p(emb), F16, S, None,
                                                       aabb6, st), "fwd")

    def timed(fn, flush):
        out = []
        for _ in range(3):
            fn()
        for _ in range(args.reps):
            if flush:
                flush_buf.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            out.append(e0.elapsed_time(e1))
        return statistics.median(out)

    def req(cnt, a=0, b=16, col=0):
        return sum(c[col] for c in cnt[a:b])

    print("\n1. footprint A/B (all 16 levels)          ms flushed  Greq/s   ms warm  Greq/s   Mreq")
    res = {}
    for name, fn, cnt, col in (("bwd T=2^19", bwd(19), c19, 0), ("bwd T=2^16", bwd(16), c16, 0),
                               ("fwd T=2^19", fwd(19), c19, 1), ("fwd T=2^16", fwd(16), c16, 1)):
        n = req(cnt, col=col)
        tf, tw = timed(fn, True), timed(fn, False)
        res[name] = (n / tf / 1e6, n / tw / 1e6)
        print(f"   {name:<36} {tf:10.3f} {res[name][0]:8.2f} {tw:9.3f} {res[name][1]:8.2f} {n / 1e6:6.1f}")
    for k in ("bwd", "fwd"):
        a, b = res[f"{k} T=2^19"], res[f"{k} T=2^16"]
        print(f"   {k}: time per request T=2^19 / T=2^16 = {b[0] / a[0]:.2f}x flushed, {b[1] / a[1]:.2f}x warm")

    print("\n2. backward level ranges, T=2^19          ms flushed  Greq/s   ms warm  Greq/s   Mreq   slice MiB")
    allf = res["bwd T=2^19"]
    ranges = [(l, l + 1) for l in range(16)] + GROUPS + [(0, 16)]
    for a, b in ranges:
        n = req(c19, a, b)
        tf, tw = timed(bwd(19, a, b), True), timed(bwd(19, a, b), False)
        sl = (lay19.offsets[b] if b < 16 else lay19.total_entries) - lay19.offsets[a]
        print(f"   levels [{a:2d}, {b:2d})                       {tf:10.3f} {n / tf / 1e6:8.2f} {tw:9.3f} "
              f"{n / tw / 1e6:8.2f} {n / 1e6:6.1f} {sl * 8 / 2 ** 20:9.1f}")
    print(f"   (all-levels launch: {allf[0]:.2f} Greq/s flushed, {allf[1]:.2f} warm)")

    if args.config == "garden16":
        print("\n3. garden16 all-levels backward, three runs of the median (ms, flushed / warm):")
        for i in range(3):
            print(f"   run {i}: {timed(bwd(19), True):.3f} / {timed(bwd(19), False):.3f}")


if __name__ == "__main__":
    main()
