"""Kernel-time breakdown of the training step (torch.profiler, CUDA activities) — run on the GPU."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import bench
from datasets.ray_utils import get_rays
from datasets.synthetic import SyntheticLego
from modules.networks import NGP
from taichi_nerfs_b200.trainer import NGPTrainer

dev = torch.device("cuda", 0)
lay, table, ws = bench.init_weights_numpy(bench.SEED)
model = NGP(scale=0.5, max_res=1024, half_opt=True).to(dev)
with torch.no_grad():
    model.pos_encoder.hash_table.copy_(torch.from_numpy(table))
ds = SyntheticLego(batch_size=bench.BATCH).to(dev)
model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
with torch.autocast("cuda", dtype=torch.float16):
    model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
trainer = NGPTrainer(model)


def step():
    b = ds[0]
    o, d = get_rays(b["direction"], b["pose"])
    return trainer.step(o, d, b["rgb"])


for _ in range(3):
    step()
torch.cuda.synchronize()
import time
t0 = time.perf_counter()
for _ in range(5):
    step()
torch.cuda.synchronize()
print("wall ms/step", (time.perf_counter() - t0) / 5 * 1e3)
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for _ in range(3):
        step()
    torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=70))
