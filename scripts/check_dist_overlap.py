"""torchrun check (N >= 2 GPUs): both multi-GPU exchanges of the graph step (the peer-memory optimizer step, the
default on one NVLink box, and the fp16 NCCL all-reduce it falls back to), each with and without the optimizer overlap,
apply the update of a single-rank trainer on the concatenated batch of all ranks; parameters and occupancy grids stay
identical on all ranks.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 scripts/check_dist_overlap.py
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from modules.networks import NGP  # noqa: E402
from oracle.train_step import make_rays  # noqa: E402   (ray generator only)
from taichi_nerfs_b200.fast_step import StaticTrainStep  # noqa: E402
from taichi_nerfs_b200.trainer import NGPTrainer  # noqa: E402

if int(os.environ.get("WORLD_SIZE", "1")) < 2:
    sys.exit("check_dist_overlap.py checks the multi-GPU step: run it under torchrun with --nproc-per-node >= 2")
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
# a one-rank group per rank for the reference trainer (new_group is collective: every rank creates every group)
solo = [dist.new_group([r]) for r in range(world)][rank]
bits = np.load(os.path.join(ROOT, "tests", "golden", "lego_bitfield.npz"))["bitfield"]
thr = 0.01 * 1024 / 3 ** 0.5
N = 4096   # rays per rank


def batch(r, k):
    """Rank r's rays, targets and marching noise of step k."""
    o, d = make_rays(N, seed=100 * r + k)
    g = torch.Generator(device="cuda").manual_seed(100 * r + k)
    return (torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), torch.rand(N, 3, device="cuda", generator=g),
            torch.rand(N, device="cuda", generator=g))


def run(overlap_opt, p2p=None, reference=False):
    torch.manual_seed(3)
    m = NGP(scale=0.5, max_res=1024, half_opt=True).cuda()
    with torch.no_grad():
        m.pos_encoder.hash_table.mul_(2e3)
        m.density_bitfield.copy_(torch.from_numpy(bits))
    tr = NGPTrainer(m, lr=1e-2, process_group=solo if reference else None, p2p_optimizer=p2p)
    n = N * world if reference else N
    fs = StaticTrainStep(tr, n, samples_per_ray_capacity=64, overlap_optimizer=overlap_opt)
    if reference:
        assert tr.world_size == 1 and tr.p2p is None and tr.grad16 is None
    elif p2p is False:
        assert tr.p2p is None and tr.grad16 is not None
    else:
        assert tr.p2p is not None, "peer-memory optimizer unavailable (CUDA IPC / peer access failed)"
    losses = []
    for k in range(4):
        if reference:   # every rank's batch, in rank order
            o, d, gt, noise = (torch.cat(parts) for parts in zip(*(batch(r, k) for r in range(world))))
        else:           # every rank renders its own shard
            o, d, gt, noise = batch(rank, k)
        losses.append(float(fs.step(o, d, gt, noise)))
        if k == 1:
            fs.flush()
            m.update_density_grid(thr, warmup=False)
    fs.flush()
    torch.cuda.synchronize()
    tr.p2p_check()
    return m, losses


m0, l0 = run(False, reference=True)   # one rank, the concatenated batch: no gradient exchange at all
runs = {"peer-memory optimizer": run(False),
        "peer-memory optimizer + overlap": run(True),            # the default at N > 1
        "fp16 NCCL fallback": run(False, p2p=False),
        "fp16 NCCL fallback + overlap": run(True, p2p=False)}
for name, (m, _) in runs.items():
    # Adam's first updates are +-lr whatever the gradient's magnitude, so an entry whose gradient sum is ~0 moves in the
    # opposite direction when the sum is rounded differently (atomic order, summation order over the ranks; fp16
    # rounding of the fallback's transport, which flips more of them): a small fraction of entries may differ by a few
    # lr, the rest agree to 2e-3
    limit = 1e-2 if name.startswith("fp16") else 2e-3
    for pa, pb in zip(m0.parameters(), m.parameters()):
        bad = float(((pa - pb).abs() > 2e-3).float().mean())
        assert bad < limit, (name, bad)
# replicas agree bit for bit: parameters and occupancy grids
for m, _ in runs.values():
    flat = torch.cat([p.detach().reshape(-1) for p in m.parameters()])
    ref = flat.clone()
    dist.broadcast(ref, 0)
    assert torch.equal(flat, ref), "parameters differ across ranks"
    g = m.density_bitfield.clone()
    gr = g.clone()
    dist.broadcast(gr, 0)
    assert torch.equal(g, gr), "occupancy bitfields differ across ranks"
if rank == 0:
    print(f"dist check ok on {world} GPUs: losses single-rank {l0} / "
          + " / ".join(f"{name} {ls}" for name, (_, ls) in runs.items()))
dist.destroy_process_group()
