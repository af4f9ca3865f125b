"""CPU (gloo, world_size 2) coverage of the N>1 path: ray sharding + one flat-gradient all-reduce +
1/world folded into Adam must reproduce the single-process update on the concatenated batch.  Compute
is done by the CPU oracle here (no GPU in this tier); the same taichi_nerfs_b200.parallel helpers are
what NGPTrainer uses on NCCL."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _model16():
    from oracle import train_step as TS
    from taichi_nerfs_b200.layout import make_hash_layout
    rng = np.random.default_rng(5)
    lay = make_hash_layout(2 ** 12, 16, 16, 512, 2)
    table = ((rng.random((lay.total_entries, 2), dtype=np.float32) * 2 - 1) * 0.1).astype(np.float32)
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    ws = [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]
    bits = np.load(os.path.join(GOLDEN, "lego_bitfield.npz"))["bitfield"]
    return TS, TS.OracleModel(lay, table, ws, bits, half=True)


N_GLOBAL = 96
LOSS_SCALE = 1024.0


def _batch():
    from oracle.train_step import make_rays
    o, d = make_rays(N_GLOBAL, seed=11)
    r = np.random.default_rng(11)
    return o, d, r.random((N_GLOBAL, 3), dtype=np.float32), r.random(N_GLOBAL, dtype=np.float32)


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["OMP_NUM_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from taichi_nerfs_b200 import parallel
    TS, model = _model16()
    o, d, gt, nz = _batch()
    b, e = parallel.shard_bounds(N_GLOBAL, rank, world)
    rgb, cache = TS.forward(model, o[b:e], d[b:e], nz[b:e])
    loss, g_table, g_mlp = TS.backward(model, cache, rgb, gt[b:e], LOSS_SCALE)
    flat = torch.from_numpy(np.concatenate([g_table, g_mlp]))
    parallel.allreduce_gradients(flat)
    found = torch.zeros(1, dtype=torch.int32)
    parallel.allreduce_found_inf(found)
    flat = flat.numpy()
    P = g_table.size
    inv = parallel.inv_grad_scale(LOSS_SCALE, world)
    # Adam consumes grad * inv: emulate by calling the oracle step with loss_scale*world
    TS.adam(model, flat[:P].copy(), flat[P:].copy(), 1e-2, LOSS_SCALE, world_size=world)
    assert abs(inv - 1.0 / (LOSS_SCALE * world)) < 1e-12 and int(found) == 0
    np.save(os.path.join(out_dir, f"table_{rank}.npy"), model.table)
    np.save(os.path.join(out_dir, f"w_{rank}.npy"), np.concatenate([w.reshape(-1) for w in model.ws]))
    dist.barrier()
    dist.destroy_process_group()


def test_shard_bounds():
    from taichi_nerfs_b200.parallel import shard_bounds
    for n, w in ((96, 2), (97, 4), (8192, 8), (5, 8)):
        cuts = [shard_bounds(n, r, w) for r in range(w)]
        assert cuts[0][0] == 0 and cuts[-1][1] == n
        assert all(cuts[i][1] == cuts[i + 1][0] for i in range(w - 1))
        sizes = [e - b for b, e in cuts]
        assert max(sizes) - min(sizes) <= 1


def test_two_rank_update_equals_single_process(tmp_path):
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    t0, t1 = np.load(tmp_path / "table_0.npy"), np.load(tmp_path / "table_1.npy")
    w0, w1 = np.load(tmp_path / "w_0.npy"), np.load(tmp_path / "w_1.npy")
    assert np.array_equal(t0, t1) and np.array_equal(w0, w1)  # replicas stay bit-identical

    # single process on the concatenated batch
    TS, model = _model16()
    before = model.table.copy()
    o, d, gt, nz = _batch()
    rgb, cache = TS.forward(model, o, d, nz)
    loss, g_table, g_mlp = TS.backward(model, cache, rgb, gt, LOSS_SCALE)
    TS.adam(model, g_table, g_mlp, 1e-2, LOSS_SCALE)
    wref = np.concatenate([w.reshape(-1) for w in model.ws])
    # mean-of-shard-means == global mean (equal shards); Adam's first step is lr*sign(g) so compare with
    # a tolerance that only forgives entries whose gradient is ~0
    moved = np.abs(model.table - before) > 0
    assert moved.any()
    assert np.mean(np.isclose(t0, model.table, rtol=0, atol=2e-4)) > 0.999
    assert np.mean(np.isclose(w0, wref, rtol=0, atol=2e-4)) > 0.999


def _worker_p2p(rank, world, port, out_dir):
    """The peer-memory optimizer step (csrc/p2p.cu, NGPTrainer._enqueue_update_p2p) with two processes on the CPU: the
    'peer buffers' are files both ranks map (np.memmap) — gradient, fp16 shadow, flag block.  No collective touches the
    gradient: rank r reads slice r of BOTH gradient buffers, sums in rank order, applies the oracle's Adam to the slice
    it owns and stores the new fp16 slice into BOTH shadow buffers; the MLP weights are updated by every rank from the
    same peer sums.  The flag barrier (epoch + inf bit per rank) is emulated with the flag file + a gloo barrier."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["OMP_NUM_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import oracle as O
    from taichi_nerfs_b200 import parallel
    TS, model = _model16()
    o, d, gt, nz = _batch()
    b, e = parallel.shard_bounds(N_GLOBAL, rank, world)
    rgb, cache = TS.forward(model, o[b:e], d[b:e], nz[b:e])
    loss, g_table, g_mlp = TS.backward(model, cache, rgb, gt[b:e], LOSS_SCALE)
    P, M = g_table.size, g_mlp.size
    total = P + M

    def peer(kind, r, dtype, n):     # rank r's buffer, mapped by everybody
        return np.memmap(os.path.join(out_dir, f"{kind}_{r}.bin"), dtype=dtype, mode="r+", shape=(n,))
    if rank == 0:
        for r in range(world):
            for kind, dtype, n in (("grad", np.float32, total), ("shadow", np.float16, total), ("flags", np.int32, world)):
                np.memmap(os.path.join(out_dir, f"{kind}_{r}.bin"), dtype=dtype, mode="w+", shape=(n,)).flush()
    dist.barrier()
    grads = [peer("grad", r, np.float32, total) for r in range(world)]
    shadows = [peer("shadow", r, np.float16, total) for r in range(world)]
    flags = [peer("flags", r, np.int32, world) for r in range(world)]
    # backward: the gradient lands in this rank's own buffer; the inf bit is raised at the source
    grads[rank][:P] = g_table
    grads[rank][P:] = g_mlp
    grads[rank].flush()
    bit = int(O.check_finite(g_table) or O.check_finite(g_mlp))
    for r in range(world):           # barrier 1: publish (epoch 1, inf bit) to every peer, wait for all of them
        flags[r][rank] = 2 * 1 + bit
        flags[r].flush()
    dist.barrier()
    mine = np.array(peer("flags", rank, np.int32, world))
    assert all(int(v) >> 1 == 1 for v in mine)
    found = int(any(int(v) & 1 for v in mine))
    assert found == 0
    lo, hi = parallel.optimizer_shard(P, rank, world)
    inv = parallel.inv_grad_scale(LOSS_SCALE, world)
    model.step += 1
    # owned table slice: peer loads, fixed rank order
    g = np.array(grads[0][lo:hi])
    for r in range(1, world):
        g = (g + np.array(grads[r][lo:hi])).astype(np.float32)
    sh = np.zeros(hi - lo, np.float16)
    O.adam_step(model.table[lo:hi], g, model.m[lo:hi], model.v[lo:hi], 1e-2, model.step, inv_scale=inv, param_f16=sh)
    for r in range(world):           # peer stores of the new fp16 slice
        shadows[r][lo:hi] = sh
        shadows[r].flush()
    # replicated MLP weights: every rank, same sums in the same order
    gm = np.array(grads[0][P:])
    for r in range(1, world):
        gm = (gm + np.array(grads[r][P:])).astype(np.float32)
    off, goff = P, 0
    for w in model.ws:
        flat = w.reshape(-1)
        O.adam_step(flat, np.ascontiguousarray(gm[goff:goff + flat.size]), model.m[off:off + flat.size],
                    model.v[off:off + flat.size], 1e-2, model.step, inv_scale=inv)
        shadows[rank][off:off + flat.size] = flat.astype(np.float16)
        off += flat.size
        goff += flat.size
    dist.barrier()                   # barrier 2: everybody has read my gradient and written my shadow
    grads[rank][:] = 0               # ... so it can be cleared
    np.save(os.path.join(out_dir, f"shadow_{rank}.npy"), np.array(peer("shadow", rank, np.float16, total)))
    np.save(os.path.join(out_dir, f"own_{rank}.npy"), model.table[lo:hi].copy())
    np.save(os.path.join(out_dir, f"w_{rank}.npy"), np.concatenate([w.reshape(-1) for w in model.ws]))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_peer_memory_optimizer_equals_replicated(tmp_path):
    """The data flow of the peer-memory optimizer step (no collective on the gradient) == the replicated update."""
    world = 2
    rep = tmp_path / "rep"
    pp = tmp_path / "p2p"
    rep.mkdir()
    pp.mkdir()
    mp.spawn(_worker, args=(world, _free_port(), str(rep)), nprocs=world, join=True)
    mp.spawn(_worker_p2p, args=(world, _free_port(), str(pp)), nprocs=world, join=True)
    t_rep = np.load(rep / "table_0.npy")
    w_rep = np.load(rep / "w_0.npy")
    P = t_rep.size
    own = np.concatenate([np.load(pp / "own_0.npy"), np.load(pp / "own_1.npy")])
    assert np.array_equal(own, t_rep)                       # the owners' fp32 slices = the replicated table
    s0, s1 = np.load(pp / "shadow_0.npy"), np.load(pp / "shadow_1.npy")
    assert np.array_equal(s0, s1)                           # both ranks hold the same fp16 shadow ...
    assert np.array_equal(s0[:P], t_rep.astype(np.float16))  # ... = the cast of the table
    assert np.array_equal(s0[P:], w_rep.astype(np.float16))
    assert np.array_equal(np.load(pp / "w_0.npy"), w_rep) and np.array_equal(np.load(pp / "w_1.npy"), w_rep)


def test_optimizer_shard_bounds():
    from taichi_nerfs_b200.parallel import optimizer_shard
    P = 11420064                                   # the stock table (SURVEY.md §8)
    for w in (2, 4, 8):
        cuts = [optimizer_shard(P, r, w) for r in range(w)]
        assert cuts[0][0] == 0 and cuts[-1][1] == P and all(a[1] == b[0] for a, b in zip(cuts, cuts[1:]))
        assert all((b - a) % 4 == 0 and a % 4 == 0 for a, b in cuts)
    with pytest.raises(ValueError):
        optimizer_shard(10, 0, 4)
