"""Time the voxel-grid model (`--model_name svox`, G = 256, degree 2) through the graph-captured step against the module
path, and its node-block optimizer pass against the dense one, on one GPU.

  python scripts/bench_voxel_step.py [--steps 200] [--rays 8192] [--spr 512] [--out bench_voxel_step.json]

Set-up of scripts/bench_voxel_grid.py: the default VoxelGrid trained for --warm module-path steps on the synthetic
scene, batches of --rays rays.  Then, without and with the regularisers (0.01, 0.01, 0):
  - NGPTrainer.step on the dataset's batches and StaticTrainStep.step_sampled (overlap_optimizer=True, capacity
    --spr rows per ray) on batches drawn from the same images, alternated, 3 windows of --steps steps each; the samples
    of the last step of every window, and the rays the graph step cut short for capacity summed over every timed step
    (one device-side add after each step, inside the graph arm's windows);
  - the finite check + Adam over the node block B (enqueue_update(voxel_block=B)) against the dense check + Adam over
    the whole flat buffer (enqueue_update()), on the same buffers.  Each is captured into a CUDA graph, so no host
    launch gap is timed (both include the two one-thread scalar launches, hyper and GradScaler update), and replayed
    after a 256 MB write that evicts the L2, median of 20, with GB/s from the bytes the two passes must move (computed
    here).
The card's name, power limit and SM clocks are read in the same process."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

REG = (0.01, 0.01, 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warm", type=int, default=500)
    ap.add_argument("--rays", type=int, default=8192)
    ap.add_argument("--spr", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_voxel_step.py measures the GPU; no CUDA device found")
    from bench_voxel_grid import card, timed
    from datasets.ray_utils import get_rays
    from modules.rendering import MAX_SAMPLES
    from modules.voxel_grid import VoxelGrid
    from taichi_nerfs_b200.fast_step import StaticTrainStep
    from taichi_nerfs_b200.trainer import NGPTrainer
    from test_gpu_e2e import _small_dataset

    dev = torch.device("cuda")
    torch.manual_seed(23)
    ds = _small_dataset(root_dir='', split='train', downsample=1.0, seed=23).to(dev)
    ds.batch_size = args.rays
    ds.ray_sampling_strategy = 'all_images'
    ds.build_image_bank()
    m = VoxelGrid().to(dev)
    m.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
    tr = NGPTrainer(m, lr=1e-2, max_steps=args.warm + 20 * args.steps)
    thr = 0.01 * MAX_SAMPLES / 3 ** 0.5
    k = 0
    last = {}

    def module_step(grid_update=False):
        nonlocal k
        data = ds[k % len(ds)]
        if grid_update and k % 16 == 0:
            with torch.autocast(device_type='cuda', dtype=torch.float16):
                m.update_density_grid(thr, warmup=k < 256)
        o, d = get_rays(data['direction'], data['pose'])
        last["module"] = tr.step(o, d, data['rgb'])[1]
        k += 1

    for _ in range(args.warm):
        module_step(grid_update=True)
    torch.cuda.synchronize()

    def window(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / args.steps

    out = {"card": card(), "G": m.field_size, "sh_degree": m.sh_degree, "params": tr.flat_param.numel(),
           "rays": args.rays, "warm_steps": args.warm, "steps_per_window": args.steps, "block": list(m._reg_block)}
    for name, reg in (("plain", None), ("reg", REG)):
        tr.voxel_reg = reg
        fs = StaticTrainStep(tr, args.rays, samples_per_ray_capacity=args.spr, overlap_optimizer=True)
        fs.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=23)
        fs.step_sampled()                           # warm the sampled graphs
        fs.flush()
        arms = {"module": [], "graph": []}
        samples = {"module": [], "graph": []}
        cut = torch.zeros((), device=dev, dtype=torch.int64)

        def graph_step():
            fs.step_sampled()
            cut.add_(fs.counter[1])

        for _ in range(3):
            arms["module"].append(window(module_step))
            samples["module"].append(int(last["module"]["rm_samples"]))
            arms["graph"].append(window(graph_step))
            samples["graph"].append(int(fs.counter[0]))
            fs.flush()
        out[name] = {
            "module_ms_windows": [round(w, 3) for w in arms["module"]],
            "graph_ms_windows": [round(w, 3) for w in arms["graph"]],
            "samples_last_step": samples, "graph_capacity_rows": fs.cap,
            "graph_rays_cut_all_timed_steps": int(cut),
            "graph_kernels_per_replay": fs.kernels_per_replay_sampled,
            "graph_faster_every_window": all(g < mm for g, mm in zip(arms["graph"], arms["module"])),
        }
        del fs
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    tr.voxel_reg = None

    # the optimizer passes alone on the trainer's buffers (with g = 0 outside B, as the graph step leaves it)
    flush = torch.zeros(64 << 20, device=dev)    # 256 MB > the 50 MB L2
    tr.found_inf.zero_()
    block = m._reg_block
    graphs = {}
    for name, kw in (("dense", {}), ("block", dict(voxel_block=block))):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            tr.enqueue_update(**kw)                  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            tr.enqueue_update(**kw)
    t_dense = timed(graphs["dense"].replay, flush)
    t_block = timed(graphs["block"].replay, flush)
    P = tr.flat_param.numel()
    nb = 1
    for a in range(3):
        nb *= block[a + 3] - block[a]
    PB = nb * (3 * m.sh_dim + 1)
    # the finite check reads the gradient; Adam reads param, grad, m, v and writes param, m, v and the zeroed gradient
    dense_bytes, block_bytes = P * 4 * 9, PB * 4 * 9
    out.update({
        "dense_check_adam_ms": round(t_dense, 4), "dense_bytes": dense_bytes,
        "dense_GBps": round(dense_bytes / (t_dense * 1e-3) / 1e9, 1),
        "block_check_adam_ms": round(t_block, 4), "block_elements": PB, "block_bytes": block_bytes,
        "block_GBps": round(block_bytes / (t_block * 1e-3) / 1e9, 1), "card_after": card(),
    })
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
