"""Config 5 of BASELINE.json: one 800x800 test-time frame (gui.py path), occupancy A (trained-Lego bitfield)."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from datasets.ray_utils import get_ray_directions, get_rays
from datasets.synthetic import SyntheticLego, hemisphere_poses
from modules.intersection import ray_aabb_intersection
from modules.networks import NGP
from modules.rendering import _render_rays_test, render

dev = torch.device("cuda", 0)
lay, table, ws = bench.init_weights_numpy(bench.SEED)
model = NGP(scale=0.5, max_res=1024, half_opt=True).to(dev)
bits = np.load(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "lego_bitfield.npz"))["bitfield"]
with torch.no_grad():
    model.pos_encoder.hash_table.copy_(torch.from_numpy(table * 2e3))
    model.density_bitfield.copy_(torch.from_numpy(bits))
ds = SyntheticLego(n_images=4)
K = ds.K.to(dev)
pose = hemisphere_poses(4)[1].to(dev)
impl = sys.argv[1] if len(sys.argv) > 1 else "loop"


def frame():
    with torch.autocast("cuda", dtype=torch.float16):
        directions = get_ray_directions(800, 800, K, device=dev)
        rays_o, rays_d = get_rays(directions, pose)
        if impl == "loop":   # the reference-shaped incremental loop
            rays_o, rays_d = rays_o.contiguous(), rays_d.contiguous()
            return _render_rays_test(model, rays_o, rays_d, ray_aabb_intersection(rays_o, rays_d, model.scale))
        return render(model, rays_o, rays_d, test_time=True)


for _ in range(3):
    r = frame()
torch.cuda.synchronize()
t0 = time.perf_counter()
n = 10
for _ in range(n):
    r = frame()
torch.cuda.synchronize()
dt = (time.perf_counter() - t0) / n
print(f"impl={impl} ms/frame={dt * 1e3:.2f} fps={1 / dt:.1f} samples/ray={float(r['total_samples']) / 640000:.2f} "
      f"opacity_mean={float(r['opacity'].mean()):.4f} rgb_mean={float(r['rgb'].mean()):.4f}")
if "--profile" in sys.argv:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            frame()
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=18, max_name_column_width=60))
