"""Time the F = 2 hash-table backward of this build against other builds of the library, on the real sample stream
of the graph-captured training step (xyzs[:S], demb[:S] after --steps steps, as scripts/hash_l2_probe.py takes it).

For each level group of the step's plan (ngp_hash_bwd_level_groups at the device's L2), the whole level range and any
--ranges, every build's ngp_hash_encode_bwd_levels is launched in turn, the L2 flushed before every launch, CUDA
events, median of --reps.  Requests per second use the lane-walk model of scripts/hash_corner_reuse.py on the first
--count-samples samples, scaled to S.  The forward (ngp_hash_encode_fwd_dyn) is timed the same way.

    python scripts/hash_bwd_builds.py --lib parent=/path/to/libngp_b200.so [--lib ...]
        [--config lego_half|garden16|lego_fp32_1024] [--steps 25] [--reps 21] [--ranges 0:6,6:11]
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
from hash_l2_probe import gpu_stream  # noqa: E402
from taichi_nerfs_b200.layout import make_hash_layout  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", choices=("lego_half", "garden16", "lego_fp32_1024"), default="lego_half")
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--count-samples", type=int, default=1 << 21)
    ap.add_argument("--ranges", default="")
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of another build")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script times kernels on the GPU")
    from taichi_nerfs_b200 import _lib
    from taichi_nerfs_b200._lib import F16, F32, check, load
    print(f"card: {card()}")
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    print(f"device: {props.name}, {props.multi_processor_count} SMs, L2 {props.L2_cache_size / 2 ** 20:.1f} MiB")
    cfg = bench.CONFIGS[args.config]
    lay = make_hash_layout(2 ** 19, 16, 16, cfg["max_res"], 2)
    cl = lay.as_ctypes()
    builds = {"this build": load()}
    for spec in args.lib:
        name, path = spec.split("=", 1)
        other = C.CDLL(os.path.abspath(path))
        for fn in ("ngp_hash_encode_bwd_levels", "ngp_hash_encode_fwd_dyn"):
            getattr(other, fn).restype, getattr(other, fn).argtypes = _lib.EXPORTS[fn]
        builds[name] = other

    xyz, demb, aabb6 = gpu_stream(args.config, args.steps)
    S = xyz.shape[0]
    tag = F16 if cfg["half"] else F32
    demb = demb.to(torch.float16 if cfg["half"] else torch.float32)
    n_cnt = min(S, args.count_samples)
    lo, span = np.asarray(aabb6[:3], np.float32), np.asarray(aabb6[3:], np.float32)
    xn = ((xyz[:n_cnt].cpu().numpy() - lo) / span).astype(np.float32)
    cnt = [hcr.count_level(lay, level, xn) for level in range(lay.levels)]
    bwd_req = [c["bwd_new"] * S / n_cnt for c in cnt]
    fwd_req = [c["old"] * S / n_cnt for c in cnt]
    print(f"{args.config}: S = {S} samples after {args.steps} steps")

    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    grad = torch.zeros(lay.total_param_size, device=dev)
    rng = torch.Generator(device=dev).manual_seed(bench.SEED)
    table = (torch.rand(lay.total_param_size, device=dev, generator=rng) * 2 - 1) * 1e-4
    table = table.half() if cfg["half"] else table
    emb = torch.empty(S, lay.out_dim, device=dev, dtype=table.dtype)
    flush_buf = torch.empty(256 << 20, device=dev, dtype=torch.uint8)

    def timed(fns):
        """launches of the functions in turn, L2 flushed before each: median ms per function"""
        out = [[] for _ in fns]
        for fn in fns:
            for _ in range(3):
                fn()
        for _ in range(args.reps):
            for i, fn in enumerate(fns):
                flush_buf.fill_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                out[i].append(e0.elapsed_time(e1))
        return [statistics.median(o) for o in out]

    groups = (C.c_int32 * 17)()
    ng = load().ngp_hash_bwd_level_groups(C.byref(cl), 0, lay.levels, props.L2_cache_size if S >= 1 << 20 else 0,
                                          groups)
    ranges = [(groups[i], groups[i + 1]) for i in range(ng)] + ([(0, lay.levels)] if ng > 1 else [])
    ranges += [tuple(int(v) for v in r.split(":")) for r in args.ranges.split(",") if r]
    print(f"\nbackward ({'fp16' if cfg['half'] else 'fp32'} dL/demb), level groups {list(groups)[: ng + 1]}")
    print(f"   {'levels':<10} {'build':<12} {'ms':>8} {'Greq/s':>7}")
    for a, b in ranges:
        fns = [lambda lib=lib, a=a, b=b: check(lib.ngp_hash_encode_bwd_levels(
            p(xyz), p(demb), tag, C.byref(cl), p(grad), S, None, aabb6, a, b, None, st), "bwd")
            for lib in builds.values()]
        req = sum(bwd_req[a:b])
        for name, t in zip(builds, timed(fns)):
            print(f"   [{a:2d}, {b:2d})   {name:<12} {t:8.4f} {req / t / 1e6:7.1f}")

    print(f"\nforward, all {lay.levels} levels")
    fns = [lambda lib=lib: check(lib.ngp_hash_encode_fwd_dyn(p(xyz), p(table), C.byref(cl), p(emb), tag, S, None,
                                                             aabb6, st), "fwd") for lib in builds.values()]
    for name, t in zip(builds, timed(fns)):
        print(f"   {name:<12} {t:8.4f} {sum(fwd_req) / t / 1e6:7.1f}")
    print(f"\ncard after the runs: {card()}")


if __name__ == "__main__":
    main()
