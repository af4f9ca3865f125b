"""Tri-plane encoder on the GPU: kernel times, training throughput against the stock hash model, one frame.

Prints one JSON line:
  gpu            name, power limit and SM clock (nvidia-smi, read in this run, the SM clock right after the kernels)
  kernels        per max_res (1024, 4096): forward and backward of the tri-plane encoder on the samples of one
                 training step (8192 Lego-shape rays marched through the reference's Lego occupancy bitfield); CUDA
                 events, L2 flushed between repeats, median of 5; algorithmic bytes per sample and GB/s
  train          module-path training rays/s (NGPTrainer.step, batch 8192) of a tri-plane and of the stock hash
                 (--half_opt) model, alternated in the same run
  frame          one 800x800 frame of the compacting renderer (FrameRenderer graph replay) of the tri-plane model

Algorithmic bytes per sample (L levels, F features, fp32): forward = 12 (xyz) + 12*L*F*4 (3 planes x 4 corners,
gathered) + L*F*4 (output); backward = 12 + L*F*4 (dL/dout) + 12*L*F*4 (recomputed gathers) + 12*L*F*4 (reduction
payload).  Cache hits are not subtracted, so GB/s is a rate of the payload the kernel moves, not of HBM traffic.

Usage: python scripts/bench_triplane.py [--steps 50] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl, sm, smax = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "error": f"nvidia-smi: {e}"}


def lego_bits():
    return np.load(os.path.join(ROOT, "tests", "golden", "lego_bitfield.npz"))["bitfield"]


def make_rays(n, seed):
    from oracle.train_step import make_rays as mk
    o, d = mk(n, seed=seed)
    return torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()


def frame_rays(w=800, h=800, focal=1111.111, radius=1.4):
    """One pinhole camera's w x h rays looking at the origin from the upper hemisphere."""
    c = np.array([0.8, -0.9, 0.75])
    c = c / np.linalg.norm(c) * radius
    fwd = -c / np.linalg.norm(c)
    right = np.cross(fwd, [0, 0, 1.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    u, v = np.meshgrid(np.arange(w), np.arange(h))
    dc = np.stack([(u - w / 2 + .5) / focal, (v - h / 2 + .5) / focal, np.ones_like(u, float)], -1).reshape(-1, 3)
    d = dc[:, :1] * right + dc[:, 1:2] * down + dc[:, 2:] * fwd
    o = np.broadcast_to(c, d.shape)
    return (torch.from_numpy(np.ascontiguousarray(o, np.float32)).cuda(),
            torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda())


def step_samples(model, n_rays=8192, seed=0):
    """The positions (in [0,1]) of one training step's march."""
    from taichi_nerfs_b200 import ops
    o, d = make_rays(n_rays, seed)
    hits = ops.ray_aabb_intersect(o, d, model.scale)
    noise = torch.rand(n_rays, device="cuda")
    counter, rays_a = ops.raymarching_train_count(o, d, hits, model.density_bitfield, noise, model.cascades,
                                                  model.scale, 0.0, model.grid_size, 1024)
    S = int(counter[0])
    xyzs = torch.empty(S, 3, device="cuda")
    dirs = torch.empty(S, 3, device="cuda")
    deltas = torch.empty(S, device="cuda")
    ts = torch.empty(S, device="cuda")
    ops.raymarching_train_write(o, d, hits, model.density_bitfield, noise, model.cascades, model.scale, 0.0,
                                model.grid_size, counter, rays_a, xyzs, dirs, deltas, ts)
    return ((xyzs - model.xyz_min) / (model.xyz_max - model.xyz_min)).contiguous()


def time_kernel(fn, reset=None, reps=5):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > 50 MB L2
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


def bench_kernels(max_res):
    from modules.networks import NGP
    from taichi_nerfs_b200 import ops
    torch.manual_seed(0)
    m = NGP(scale=0.5, pos_encoder_type="triplane", max_res=max_res).cuda()
    m.density_bitfield.copy_(torch.from_numpy(lego_bits()))
    enc = m.pos_encoder
    x = step_samples(m)
    S = x.shape[0]
    tab, cl = enc.plane_embedding.detach(), enc._clayout
    L, F = enc.levels, enc.feature_per_level
    out = ops.triplane_encode_fwd(x, tab, cl)
    dout = torch.randn_like(out)
    grad = torch.zeros(enc.total_param_size, device="cuda")
    t_f = time_kernel(lambda: ops.triplane_encode_fwd(x, tab, cl, out=out))
    t_b = time_kernel(lambda: ops.triplane_encode_bwd(x, tab, dout, cl, grad), reset=grad.zero_)
    b_f = 12 + 12 * L * F * 4 + L * F * 4
    b_b = 12 + L * F * 4 + 2 * 12 * L * F * 4
    return {"max_res": max_res, "samples": S, "fwd_ms": t_f, "bwd_ms": t_b, "fwd_bytes_per_sample": b_f,
            "bwd_bytes_per_sample": b_b, "fwd_GBps": b_f * S / t_f / 1e6, "bwd_GBps": b_b * S / t_b / 1e6}


def make_trainer(kind):
    from modules.networks import NGP
    from taichi_nerfs_b200.trainer import NGPTrainer
    torch.manual_seed(0)
    if kind == "triplane":
        m = NGP(scale=0.5, pos_encoder_type="triplane", max_res=1024).cuda()
    else:
        m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    m.density_bitfield.copy_(torch.from_numpy(lego_bits()))
    return m, NGPTrainer(m, lr=1e-2, max_steps=100000)


def bench_train(steps, rounds, batch=8192):
    arms = {k: make_trainer(k) for k in ("triplane", "hash")}
    data = [(*make_rays(batch, s), torch.rand(batch, 3, device="cuda")) for s in range(8)]
    res = {k: [] for k in arms}
    for k, (_, tr) in arms.items():           # warm-up
        for i in range(5):
            tr.step(*data[i % 8])
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, (_, tr) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                tr.step(*data[i % 8])
            torch.cuda.synchronize()
            res[k].append(batch * steps / (time.perf_counter() - t0))
    return {k: {"rays_per_s_median": float(np.median(v)), "rays_per_s": v} for k, v in res.items()}, arms


def bench_frame(model):
    from taichi_nerfs_b200.render_frame import FrameRenderer
    o, d = frame_rays()
    fr = FrameRenderer(model, o.shape[0])
    for _ in range(2):
        out = fr.render(o, d)
    times = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fr.render(o, d)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return {"rays": o.shape[0], "ms_median": float(np.median(times)), "ms": times,
            "samples": int(out["total_samples"]), "rounds": fr.rounds_run,
            "opacity_mean": float(out["opacity"].mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_triplane.py needs a CUDA device")
    from taichi_nerfs_b200 import _lib
    _lib.load()
    result = {"gpu": gpu_info()}
    result["kernels"] = [bench_kernels(r) for r in (1024, 4096)]
    result["gpu"]["sm_clock_after_kernels"] = gpu_info().get("sm_clock")
    train, arms = bench_train(args.steps, args.rounds)
    result["train"] = train
    result["frame"] = bench_frame(arms["triplane"][0])
    result["note"] = ("random-init models on the reference's trained Lego occupancy bitfield; train rays from random "
                      "cameras on the Lego hemisphere; the frame renders the trained tri-plane arm on the same bitfield")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
