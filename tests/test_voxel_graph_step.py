"""Argument validation of the voxel-grid graph step's C-ABI entries (ngp_voxel_bwd_dyn, ngp_check_finite_voxel_block,
ngp_adam_step_voxel_block_dyn); none of them needs a GPU to refuse bad arguments."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def _b6(*v):
    return (C.c_int32 * 6)(*v)


def test_block_entries_validate_their_arguments(lib):
    buf = (C.c_float * 64)()
    p = C.c_void_p(C.addressof(buf))
    flag = (C.c_int32 * 1)()
    f = C.c_void_p(C.addressof(flag))
    ok = _b6(0, 0, 0, 2, 2, 2)
    chk = lambda *a: lib.ngp_check_finite_voxel_block(*a)                                      # noqa: E731
    adam = lambda g, c, b, *ptrs: lib.ngp_adam_step_voxel_block_dyn(*ptrs, g, c, b, None, p, 0.9, 0.999, 1e-15,  # noqa
                                                                   None)
    for bad in (_b6(-1, 0, 0, 2, 2, 2), _b6(0, 0, 0, 3, 2, 2), _b6(1, 0, 0, 1, 2, 2), _b6(0, 2, 0, 2, 1, 2),
                _b6(0, 0, 0, 2, 2, 0)):
        assert chk(p, 2, 1, bad, f, None) != 0
        assert b"lo < hi" in lib.ngp_last_error()
        assert adam(2, 1, bad, p, p, p, p) != 0
    assert chk(p, 2, 1, None, f, None) != 0 and adam(2, 1, None, p, p, p, p) != 0
    assert chk(p, 2, 0, ok, f, None) != 0 and adam(2, 0, ok, p, p, p, p) != 0         # C >= 1
    assert chk(p, 0, 1, ok, f, None) != 0 and adam(0, 1, ok, p, p, p, p) != 0         # G >= 1
    assert chk(None, 2, 1, ok, f, None) != 0 and chk(p, 2, 1, ok, None, None) != 0
    for k in range(4):
        ptrs = [p] * 4
        ptrs[k] = None
        assert adam(2, 1, ok, *ptrs) != 0, k
    assert lib.ngp_adam_step_voxel_block_dyn(p, p, p, p, 2, 1, ok, None, None, 0.9, 0.999, 1e-15, None) != 0  # hyper


def test_bwd_dyn_validates_its_arguments(lib):
    from taichi_nerfs_b200.layout import make_voxel_layout
    lay = make_voxel_layout(4, 0.25, 2).as_ctypes()
    buf = (C.c_float * 64)()
    p = C.c_void_p(C.addressof(buf))
    call = lambda *a: lib.ngp_voxel_bwd_dyn(*a)                                                # noqa: E731
    ok = [p, p, p, p, p, p, C.byref(lay), p, p]
    assert call(*ok, 0, None, None, None) == 0                   # n_max == 0: nothing to launch
    assert call(*ok, -1, None, None, None) != 0
    for k in (0, 1, 2, 3, 4, 5, 7, 8):
        args = list(ok)
        args[k] = None
        assert call(*args, 8, None, None, None) != 0, k
    bad = make_voxel_layout(4, 0.25, 2).as_ctypes()
    bad.sh_degree = 3
    assert call(*ok[:6], C.byref(bad), p, p, 8, None, None, None) != 0
    assert b"sh_degree" in lib.ngp_last_error()
    # the static entry keeps refusing an unknown mapping before delegating
    assert lib.ngp_voxel_bwd(*ok, 1, None, 2, None) != 0 and b"mapping" in lib.ngp_last_error()

