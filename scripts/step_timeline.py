"""Real (concurrent, warm) GPU timeline of the graph-captured training step: kernel start / end stamps from CUPTI via
torch.profiler, for a few steady-state replays.  Prints, per step: the span (first kernel start -> last kernel end), the
summed kernel time on the critical stream, the gaps between consecutive kernels, and the overlap of the optimizer branch
with the marching branch.  Run on the GPU:  python scripts/step_timeline.py [out.txt]"""
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

import bench
from datasets.synthetic import SyntheticLego
from modules.networks import NGP
from taichi_nerfs_b200.fast_step import StaticTrainStep
from taichi_nerfs_b200.trainer import NGPTrainer

dev = torch.device("cuda", 0)
cfg = bench.CONFIGS["lego_half"]
lay, table, ws = bench.init_weights_numpy(bench.SEED)
model = NGP(scale=0.5, max_res=1024, half_opt=True).to(dev)
with torch.no_grad():
    model.pos_encoder.hash_table.copy_(torch.from_numpy(table))
    for p, w in zip(bench.mlp_params(model), ws):
        p.copy_(torch.from_numpy(w))
ds = SyntheticLego(batch_size=bench.BATCH, seed=bench.SEED).to(dev)
model.mark_invisible_cells(ds.K, ds.poses, ds.img_wh)
model.update_density_grid(bench.DENSITY_THRESHOLD, warmup=True)
trainer = NGPTrainer(model)
fast = StaticTrainStep(trainer, bench.BATCH, samples_per_ray_capacity=384, overlap_optimizer=True)
ds.build_image_bank()
fast.attach_ray_source(ds.rays, ds.poses, ds.directions, seed=bench.SEED)
for _ in range(30):
    fast.step_sampled()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(50):
    fast.step_sampled()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 50
S = int(fast.counter[0])
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(6):
        fast.step_sampled()
    torch.cuda.synchronize()
path = os.path.join(tempfile.gettempdir(), "trace.json")
prof.export_chrome_trace(path)
ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
ev.sort(key=lambda e: e["ts"])
out = [f"graph step, S = {S} samples, {ms:.4f} ms/step by CUDA events over 50 back-to-back replays (no grid update)"]
# split into steps at the sampler kernel
starts = [i for i, e in enumerate(ev) if "sample_ray_batch" in e["name"]]
for a, b in zip(starts[2:-1], starts[3:]):
    step = ev[a:b]
    t0 = step[0]["ts"]
    span = max(e["ts"] + e["dur"] for e in step) - t0
    out.append(f"--- step: span {span:.1f} us (next step starts {ev[b]['ts'] - t0:.1f} us after this one)")
    prev_end = None
    busy = 0.0
    for e in step:
        gap = "" if prev_end is None else f"gap {e['ts'] - prev_end:6.1f}"
        out.append(f"  +{e['ts'] - t0:8.1f} us  dur {e['dur']:7.1f}  stream {e['args'].get('stream', '?'):>3}  {gap:12s} {e['name'][:60]}")
        prev_end = max(prev_end or 0, e["ts"] + e["dur"])
    # union of busy intervals
    iv = sorted((e["ts"], e["ts"] + e["dur"]) for e in step)
    cur_s, cur_e = iv[0]
    for s, t in iv[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, t
        else:
            cur_e = max(cur_e, t)
    busy += cur_e - cur_s
    out.append(f"  GPU busy (union of kernels) {busy:.1f} us, idle inside the step {span - busy:.1f} us")
text = "\n".join(out)
print(text)
if len(sys.argv) > 1:
    open(sys.argv[1], "w").write(text + "\n")
