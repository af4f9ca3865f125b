"""Counts, per hash-grid level, what the F = 2 hash kernels issue on a real sample stream: cell runs, forward gathers
(load instructions) and backward atomics (red requests) per sample, under two rules:

  old  every new cell gathers / flushes all 8 corners;
  new  when the new cell is a neighbour of the previous one (every per-axis delta in {-1, 0, 1}), the corners the two
       cells share are carried in registers: the backward flushes only the corners that leave (what hash_bwd_kernel
       does), and a forward that carried them would gather only the others (hash_fwd_kernel does not: DESIGN.md §4).

Both rules merge the x-neighbour pair (c, c + 1) into one load / one `red.v4` when the two entry indices differ only in
bit 0 and both corners are moved.  The lane mapping is the kernels' (hash.cu): each lane walks 16 consecutive samples
at one level, and the first sample of a chunk always starts a fresh cell.  Pure integer arithmetic on the positions;
the backward's skip of rows whose dL/dout is zero is not modelled (every row counts).

    python scripts/hash_corner_reuse.py                 # CPU: oracle forward() of the lego_half workload
    python scripts/hash_corner_reuse.py --source gpu    # GPU: xyzs[:counter[0]] of the graph-captured step
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

CHUNK = 16
M32 = np.uint64(0xFFFFFFFF)
BITS = np.array([[(c >> d) & 1 for d in range(3)] for c in range(8)], np.int64)   # [corner, axis]


def corner_indices(lay, level, g):
    """[R, 8] uint64 entry indices of the corners of cells g [R, 3] (hash.cu corner_indices, uint32 arithmetic)."""
    off, size = np.uint64(lay.offsets[level]), np.uint64(lay.map_sizes[level])
    res = np.uint64(lay.resolutions[level])
    gu = g.astype(np.uint64)
    cg = (gu[:, None, :] + BITS[None].astype(np.uint64)) & M32                        # [R, 8, 3]
    if level < lay.begin_fast_hash_level:
        h = (cg[..., 0] + cg[..., 1] * res + cg[..., 2] * ((res * res) & M32)) & M32
        h = np.where(h >= size, h - size, h)
        h = np.where(h >= size, h % size, h)
    else:
        h = cg[..., 0] ^ ((cg[..., 1] * np.uint64(2654435761)) & M32) ^ ((cg[..., 2] * np.uint64(805459861)) & M32)
        h = h & (size - np.uint64(1)) if (lay.map_sizes[level] & (lay.map_sizes[level] - 1)) == 0 else h % size
    return off + h


def moved_requests(idx, moved):
    """Requests to move the `moved` corners [R, 8] bool of cells with indices idx [R, 8]: one per x-pair whose two
    corners both move and share an aligned 2-entry block, else one per moved corner."""
    n = np.zeros(idx.shape[0], np.int64)
    for c in range(0, 8, 2):
        both = moved[:, c] & moved[:, c + 1]
        merged = both & ((idx[:, c] ^ idx[:, c + 1]) == 1)
        n += np.where(merged, 1, moved[:, c].astype(np.int64) + moved[:, c + 1])
    return n


def count_level(lay, level, xn):
    scale = np.float32(lay.scales[level])
    g = np.floor(xn * scale + np.float32(0.5)).astype(np.int64)                       # hash.cu grid_pos (fp32, no FMA)
    n = g.shape[0]
    first = np.arange(n) % CHUNK == 0
    start = first.copy()
    start[1:] |= np.any(g[1:] != g[:-1], axis=1)
    runs = np.flatnonzero(start)
    gr = g[runs]
    idx = corner_indices(lay, level, gr)
    all8 = np.ones((runs.size, 8), bool)
    full = moved_requests(idx, all8)                                                   # old rule: gather / flush all 8

    # the run that follows run r inside the same chunk (if any) and its offset to r's cell
    cont = np.zeros(runs.size, bool)                                                   # run r continues run r - 1
    cont[1:] = ~first[runs[1:]]
    delta = np.zeros_like(gr)
    delta[1:] = gr[1:] - gr[:-1]
    nb = cont & np.all(np.abs(delta) <= 1, axis=1)
    dpos, dneg = (delta == 1)[:, None, :], (delta == -1)[:, None, :]                 # [R, 1, 3]
    b = BITS[None].astype(bool)                                                        # [1, 8, 3]
    # corner c' of the new cell is corner c' + delta of the old one: carried when that lies in {0, 1}^3
    carried = nb[:, None] & ~np.any((dpos & b) | (dneg & ~b), axis=2)                 # [R, 8] new-cell corners
    # corner c of the old cell stays when c - delta lies in {0, 1}^3
    stays = ~np.any((dpos & ~b) | (dneg & b), axis=2)                                  # [R, 8], for the run r - 1
    gathers_new = moved_requests(idx, ~carried)

    leaves = np.ones((runs.size, 8), bool)                                             # corners of run r flushed at its end
    nxt = np.flatnonzero(nb[1:])                                                       # run r + 1 is a neighbour of r
    leaves[nxt] = ~stays[nxt + 1]
    atomics_new = moved_requests(idx, leaves)
    return dict(res=lay.resolutions[level], dense=level < lay.begin_fast_hash_level, runs=runs.size,
                neighbour=int(nb.sum()), changes=int(cont.sum()), old=int(full.sum()), fwd_new=int(gathers_new.sum()),
                bwd_new=int(atomics_new.sum()))


def report(lay, xn, label):
    n = xn.shape[0]
    rows = [count_level(lay, l, xn) for l in range(lay.levels)]
    print(f"{label}: {n} samples, {lay.levels} levels, {CHUNK}-sample lane chunks")
    print(f"{'lvl':>3} {'res':>5} {'kind':>6} {'changes/s':>9} {'nbr%':>6} {'old req/s':>9} "
          f"{'fwd new':>8} {'fwd cut':>7} {'bwd new':>8} {'bwd cut':>7}")
    tot = dict(old=0, fwd_new=0, bwd_new=0, changes=0)
    for l, r in enumerate(rows):
        for k in tot:
            tot[k] += r[k]
        nbp = 100.0 * r["neighbour"] / max(r["changes"], 1)
        print(f"{l:>3} {r['res']:>5} {'dense' if r['dense'] else 'hashed':>6} {r['changes'] / n:9.3f} {nbp:6.1f} "
              f"{r['old'] / n:9.3f} {r['fwd_new'] / n:8.3f} {1 - r['fwd_new'] / r['old']:7.1%} "
              f"{r['bwd_new'] / n:8.3f} {1 - r['bwd_new'] / r['old']:7.1%}")
    print(f"all levels: cell changes {tot['changes'] / n:.2f}/sample; gathers {tot['old'] / n:.2f} -> "
          f"{tot['fwd_new'] / n:.2f}/sample ({1 - tot['fwd_new'] / tot['old']:.1%} fewer); atomics "
          f"{tot['old'] / n:.2f} -> {tot['bwd_new'] / n:.2f}/sample ({1 - tot['bwd_new'] / tot['old']:.1%} fewer)")


def cpu_stream(n_rays):
    bench.host_threads()
    cfg = bench.CONFIGS["lego_half"]
    TS, model, batch = bench.oracle_workload(cfg, n_rays, bench.SEED)
    o, d, noise, _ = batch(0)
    _, cache = TS.forward(model, o, d, noise)
    return model.layout, cache["xn"], f"CPU oracle forward, lego_half, {n_rays} rays (random init, occupancy B)"


def gpu_stream(steps):
    import torch
    from datasets.synthetic import SyntheticLego
    from modules.networks import NGP
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    dev = torch.device("cuda", 0)
    cfg = bench.CONFIGS["lego_half"]
    torch.manual_seed(bench.SEED)
    lay, table, ws = bench.init_weights_numpy(bench.SEED, cfg["max_res"], cfg["half"])
    model = NGP(scale=cfg["scale"], max_res=cfg["max_res"], half_opt=True).to(dev)
    with torch.no_grad():
        model.pos_encoder.hash_table.copy_(torch.from_numpy(table).view_as(model.pos_encoder.hash_table))
        for p, w in zip(bench.mlp_params(model), ws):
            p.copy_(torch.from_numpy(w))
    ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED, img_wh=cfg["img_wh"], focal=cfg["focal"],
                       radius=cfg["radius"]).to(dev)
    model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=20000)
    fast = StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=cfg["cap"])
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
    xyz = fast.xyzs[:S].cpu().numpy()
    lo = np.asarray(fast.aabb6[:3], np.float32)
    span = np.asarray(fast.aabb6[3:], np.float32)
    return lay, ((xyz - lo) / span).astype(np.float32), f"GPU graph-captured step {steps}, lego_half, {bench.BATCH} rays"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--source", choices=("cpu", "gpu"), default="cpu")
    ap.add_argument("--rays", type=int, default=bench.BATCH, help="cpu: rays of the oracle batch")
    ap.add_argument("--steps", type=int, default=25, help="gpu: training steps before the stream is read")
    args = ap.parse_args()
    lay, xn, label = cpu_stream(args.rays) if args.source == "cpu" else gpu_stream(args.steps)
    report(lay, xn, label)


if __name__ == "__main__":
    main()
