"""Mesh export timing on the teacher Lego (DESIGN.md §6g): per-stage device time at N = 256, 512, 1024, achieved
bandwidth of each marching-cubes kernel, and peak device memory of the whole extraction.

    python scripts/bench_mesh.py [--sizes 256 512 1024] [--runs 5]

Each stage is timed with CUDA events around its launches, median of --runs runs after one warm-up run.  Bytes are the
least traffic the kernel needs, computed from the shapes: every lattice value read once (count, emit), the tile
counts and offsets, and what the kernel writes.  They are compared with the H100 SXM's 3.35 TB/s of HBM3.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, runs):
    """Median device milliseconds of fn() over `runs` runs, after one warm-up run."""
    fn()
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def bench(model, n, threshold, runs):
    from taichi_nerfs_b200 import ops
    from taichi_nerfs_b200.mesh import density_lattice, extract_mesh, vertex_colors
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    mesh = extract_mesh(model, n, threshold)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    nv, nf = len(mesh.vertices), len(mesh.faces)
    del mesh

    res = {"n": n, "vertices": nv, "faces": nf, "peak_mem_gb": peak / 1e9}
    lattice = [None]

    def fill():
        lattice[0] = None
        lattice[0] = density_lattice(model, n)
    res["lattice_fill_ms"] = timed(fill, runs)
    st = ops.McStages(lattice[0], threshold, model.scale)
    res["count_ms"] = timed(st.count, runs)
    res["scan_ms"] = timed(st.scan, runs)
    assert st.sizes() == (nv, nf)
    v = torch.empty(nv, 3, device=dev)
    nrm = torch.empty(nv, 3, device=dev)
    f = torch.empty(nf, 3, device=dev, dtype=torch.int32)
    res["emit_vertices_ms"] = timed(lambda: st.emit_vertices(nv, v, nrm), runs)
    res["emit_faces_ms"] = timed(lambda: st.emit_faces(nf, f), runs)
    res["colors_ms"] = timed(lambda: vertex_colors(model, v, nrm), runs)

    nodes = n ** 3
    tiles = -(-nodes // 1024)
    owners = min(nodes, nv)              # at most one vbase write per vertex
    traffic = {
        "count": nodes * 4 + tiles * 8,
        "scan": tiles * (8 + 16) + 2 * (-(-tiles // 1024)) * 16,
        "emit_vertices": nodes * 4 + tiles * 16 + nv * 24 + owners * 4,
        "emit_faces": nodes * 4 + tiles * 16 + nf * 12 + nf * 3 * 4,
    }
    for k, b in traffic.items():
        ms = res[f"{k}_ms"]
        res[f"{k}_bytes"] = b
        res[f"{k}_tb_per_s"] = b / (ms * 1e-3) / 1e12
        res[f"{k}_share_of_hbm"] = b / (ms * 1e-3) / HBM_BYTES_PER_S
    del st, lattice[0], v, nrm, f
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--threshold", type=float, default=10.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh.py measures on a CUDA device; there is no CPU arm")
    import __graft_entry__ as g
    from datasets.teacher import load_teacher
    if not g.stage_lego_fixture():
        raise SystemExit("the teacher Lego could not be staged")
    model = load_teacher(torch.device("cuda", 0))
    name, power = card()
    for n in args.sizes:
        r = bench(model, n, args.threshold, args.runs)
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
