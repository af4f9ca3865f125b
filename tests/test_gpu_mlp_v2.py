"""GPU: the fused MLP kernels (csrc/mlp.cu) at the sizes and entry points the training step uses.  The test names
keep the history of the project: "v1" / "v2" are now the two code paths each kernel has — the forward's fp32- and
fp16-embedding instantiations (bit for bit on fp16-representable inputs), the backward recomputing the forward vs
restarting from the activations the forward saved."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _weights(rng):
    shapes = [(64, 32), (16, 64), (64, 32), (64, 64), (3, 64)]
    return [(rng.uniform(-1, 1, s) * np.sqrt(6 / (s[0] + s[1]))).astype(np.float32) for s in shapes]


@pytest.mark.parametrize("n", [128, 129, 1000, 4096, 70001, 300 * 128 * 2 + 77])
def test_mlp_fwd_v2_equals_v1_bitwise(n):
    """fp32 embeddings holding fp16 values (v1) against the same values as fp16 (v2): identical MMA operands."""
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(n)
    emb = T(rng.standard_normal((n, 32)).astype(np.float16))
    dirs = T(rng.standard_normal((n, 3)).astype(np.float32))
    ws = [T(w) for w in _weights(rng)]
    s1, r1, sv1 = ops.mlp_fwd(emb.float(), dirs, ws, with_save=True)
    s2, r2, sv2 = ops.mlp_fwd(emb, dirs, ws, with_save=True)
    torch.cuda.synchronize()
    assert torch.equal(s1, s2)
    assert torch.equal(r1, r2)
    assert torch.equal(sv1, sv2)
    # and without the save buffer
    s3, r3 = ops.mlp_fwd(emb, dirs, ws)
    assert torch.equal(s1, s3) and torch.equal(r1, r3)


def test_mlp_fwd_v2_matches_oracle(oracle):
    from taichi_nerfs_b200 import ops
    n = 20000
    rng = np.random.default_rng(5)
    emb = rng.standard_normal((n, 32)).astype(np.float16)
    dirs = rng.standard_normal((n, 3)).astype(np.float32)
    ws = _weights(rng)
    sig_ref, rgb_ref = oracle.mlp_fwd(emb, dirs, ws)
    sig, rgb = ops.mlp_fwd(T(emb), T(dirs), [T(w) for w in ws])
    sig, rgb = sig.cpu().numpy(), rgb.float().cpu().numpy()
    # per-element fp16 flip model (tests/mlp_tolerance.py): rigorous bound on every element, 99 % within 2 ulp16(h0)
    from mlp_tolerance import check_sigma
    check_sigma(sig, sig_ref, emb, ws)
    assert np.abs(rgb - rgb_ref.astype(np.float32)).max() <= 2e-3


def test_mlp_fwd_v2_device_side_count():
    """n read from device memory (graph-captured step): rows >= *n_dev are left untouched."""
    from taichi_nerfs_b200 import _lib, ops
    lib = _lib.load()
    cap, n = 5000, 3333
    rng = np.random.default_rng(9)
    emb = T(rng.standard_normal((cap, 32)).astype(np.float16))
    dirs = T(rng.standard_normal((cap, 3)).astype(np.float32))
    ws = [T(w) for w in _weights(rng)]
    s_ref, r_ref = ops.mlp_fwd(emb[:n].contiguous(), dirs[:n].contiguous(), ws)
    sig = torch.full((cap,), -7.0, device=DEV)
    rgb = torch.full((cap, 3), -7.0, device=DEV, dtype=torch.float16)
    n_dev = torch.tensor([n], device=DEV, dtype=torch.int32)
    st, keep = ops._mlp_weights(ws)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(lib.ngp_mlp_fwd_dyn(p(emb), _lib.F16, p(dirs), C.byref(st), p(sig), p(rgb), None, cap, p(n_dev),
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert torch.equal(sig[:n], s_ref) and torch.equal(rgb[:n], r_ref)
    assert bool((sig[n:] == -7.0).all()) and bool((rgb[n:] == -7.0).all())


@pytest.mark.parametrize("n", [128, 129, 5000, 148 * 3 * 128 + 1, 300 * 128 * 2 + 77])
def test_mlp_bwd_v2_equals_v1(n):
    """Backward restarting from the saved activations (v2) against recomputing the whole forward (v1): the saved h and
    fp16 rgb are exactly what the recompute produces, so dL/dE is bit-identical; the weight gradients are per-CTA
    register sums flushed with fp32 atomics, whose order may differ between launches."""
    from taichi_nerfs_b200 import ops
    rng = np.random.default_rng(n)
    emb = T(rng.standard_normal((n, 32)).astype(np.float16))
    dirs = T(rng.standard_normal((n, 3)).astype(np.float32))
    ws = [T(w) for w in _weights(rng)]
    dsig = T((rng.standard_normal(n) * 1e-2).astype(np.float32))
    drgb = T((rng.standard_normal((n, 3)) * 1e-2).astype(np.float16))
    _, _, save = ops.mlp_fwd(emb, dirs, ws, with_save=True)
    de1, gw1 = ops.mlp_bwd(emb, dirs, ws, dsig, drgb)
    de2, gw2 = ops.mlp_bwd(emb, dirs, ws, dsig, drgb, save=save)
    de3, gw3 = ops.mlp_bwd(emb, dirs, ws, dsig, drgb, save=save)     # a second launch: no state left behind
    torch.cuda.synchronize()
    assert torch.equal(de1, de2) and torch.equal(de2, de3)
    scale = float(gw1.abs().max())
    assert float((gw1 - gw2).abs().max()) <= 2e-5 * scale
    assert float((gw2 - gw3).abs().max()) <= 2e-5 * scale
