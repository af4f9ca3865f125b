"""Camera extrinsics refinement (--extrinsics_lr, DESIGN.md §6i) without a GPU: the option's refusals, the fp64
restatement of Exp and the left Jacobian of SO(3) against central differences (theta -> 0 included), the package's
Rodrigues for the exported poses against it, and the C-ABI argument checks of the new entries."""
import ctypes as C

import numpy as np
import pytest

from pose_ref import hat, so3_exp, so3_jl, so3_log


# ---- opt.py ---------------------------------------------------------------------------------------------------------
def _opts(*args):
    from opt import get_opts
    return get_opts(list(args))


def test_extrinsics_lr_default_is_off():
    assert _opts().extrinsics_lr == 0.0
    assert _opts('--extrinsics_lr', '1e-3').extrinsics_lr == 1e-3


@pytest.mark.parametrize("v", ["-1e-3", "nan", "inf"])
def test_extrinsics_lr_must_be_finite_and_non_negative(v, capsys):
    with pytest.raises(SystemExit):
        _opts(f'--extrinsics_lr={v}')
    assert "--extrinsics_lr must be finite and >= 0" in capsys.readouterr().err


@pytest.mark.parametrize("flags, what", [(('--model_name', 'svox'), "svox"),
                                         (('--encoder_type', 'triplane'), "triplane")])
def test_extrinsics_lr_refuses_encoders_without_a_position_gradient(flags, what, capsys):
    with pytest.raises(SystemExit):
        _opts('--extrinsics_lr', '1e-3', *flags)
    err = capsys.readouterr().err
    assert what in err and "gradient wrt the sample positions" in err
    _opts('--extrinsics_lr', '0', *flags)   # off: accepted


@pytest.mark.parametrize("lr", ["0", "-1e-2", "nan", "inf"])
def test_extrinsics_lr_needs_a_positive_model_lr(lr, capsys):
    with pytest.raises(SystemExit):
        _opts('--extrinsics_lr', '1e-3', f'--lr={lr}')
    assert "needs a finite --lr > 0" in capsys.readouterr().err
    _opts('--extrinsics_lr', '0', f'--lr={lr}')   # off: --lr is not read by it


# ---- Exp and J_l against central differences -------------------------------------------------------------------------
ANGLES = [0.0, 1e-9, 1e-6, 1e-4, 9.9e-4, 1.1e-3, 1e-2, 0.3, 1.0, 2.5]


def _dirs(seed):
    v = np.random.default_rng(seed).standard_normal(3)
    return v / np.linalg.norm(v)


@pytest.mark.parametrize("theta", ANGLES)
def test_exp_is_a_rotation_matching_the_matrix_exponential(theta):
    from scipy.linalg import expm
    w = theta * _dirs(1)
    E = so3_exp(w)
    assert np.abs(E - expm(hat(w))).max() < 1e-14
    assert np.abs(E @ E.T - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(E) - 1) < 1e-14
    if theta > 1e-6:
        assert np.abs(so3_log(E) - w).max() < 1e-12


@pytest.mark.parametrize("theta", ANGLES)
def test_left_jacobian_against_central_differences(theta):
    """Exp(w + h e_k) Exp(w)^T = Exp(J_l(w) h e_k + O(h^2)): column k of J_l is the central difference of the log."""
    w = theta * _dirs(2)
    h = 1e-6
    J = np.empty((3, 3))
    E0 = so3_exp(w)
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        J[:, k] = (so3_log(so3_exp(w + e) @ E0.T) - so3_log(so3_exp(w - e) @ E0.T)) / (2 * h)
    assert np.abs(J - so3_jl(w)).max() < 1e-8, (theta, J, so3_jl(w))


@pytest.mark.parametrize("theta", ANGLES)
def test_rotation_gradient_through_the_left_jacobian(theta):
    """d/dw of g . Exp(w) R c = J_l(w)^T (d' x g), d' = Exp(w) R c: the rule the pose kernels implement."""
    rng = np.random.default_rng(3)
    w = theta * _dirs(4)
    R = so3_exp(rng.standard_normal(3))
    c, g = rng.standard_normal(3), rng.standard_normal(3)
    f = lambda v: g @ (so3_exp(v) @ R @ c)   # noqa: E731
    h = 1e-6
    num = np.array([(f(w + h * np.eye(3)[k]) - f(w - h * np.eye(3)[k])) / (2 * h) for k in range(3)])
    d = so3_exp(w) @ R @ c
    assert np.abs(num - so3_jl(w).T @ np.cross(d, g)).max() < 1e-8


def test_package_rodrigues_matches_the_restatement():
    from taichi_nerfs_b200.extrinsics import so3_exp_np
    rng = np.random.default_rng(5)
    for theta in ANGLES:
        w = theta * _dirs(int(theta * 1e6) % 97)
        assert np.abs(so3_exp_np(w[None])[0] - so3_exp(w)).max() < 1e-15
    W = rng.standard_normal((7, 3))
    assert np.abs(so3_exp_np(W) - np.stack([so3_exp(v) for v in W])).max() < 1e-15


# ---- C-ABI argument checks (no launch) ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def test_pose_argument_validation_needs_no_gpu(lib):
    from taichi_nerfs_b200._lib import F32
    from taichi_nerfs_b200.layout import make_hash_layout
    fake, odd = C.c_void_p(0x10000), C.c_void_p(0x10004)
    # pose apply: negative count, no images, null pointers, misaligned corrections; n = 0 is a no-op
    assert lib.ngp_pose_apply(fake, fake, fake, fake, 4, fake, fake, -1, None) < 0
    assert lib.ngp_pose_apply(fake, fake, fake, fake, 0, fake, fake, 8, None) < 0
    assert b"n_img" in lib.ngp_last_error()
    assert lib.ngp_pose_apply(fake, None, fake, fake, 4, fake, fake, 8, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert lib.ngp_pose_apply(fake, fake, fake, odd, 4, fake, fake, 8, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert lib.ngp_pose_apply(None, None, None, None, 4, None, None, 0, None) == 0
    # pose gradient
    assert lib.ngp_pose_grad(fake, fake, fake, fake, fake, -1, None, 8, 4, fake, None, None) < 0
    assert lib.ngp_pose_grad(fake, fake, fake, fake, fake, 8, None, -1, 4, fake, None, None) < 0
    assert lib.ngp_pose_grad(fake, fake, fake, fake, fake, 8, None, 8, 0, fake, None, None) < 0
    assert lib.ngp_pose_grad(fake, fake, fake, fake, fake, 8, None, 8, 4, None, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert lib.ngp_pose_grad(None, None, fake, fake, fake, 8, None, 8, 4, fake, None, None) < 0
    assert lib.ngp_pose_grad(None, None, None, None, None, 0, None, 0, 4, None, None, None) == 0
    # pose Adam
    assert lib.ngp_pose_adam(fake, fake, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, -1, None) < 0
    assert lib.ngp_pose_adam(fake, fake, fake, fake, None, None, 0.1, 0.9, 0.999, 1e-15, 4, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert lib.ngp_pose_adam(fake, odd, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, 4, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    for r in (-0.1, float("inf"), float("nan")):
        assert lib.ngp_pose_adam(fake, fake, fake, fake, None, fake, r, 0.9, 0.999, 1e-15, 4, None) < 0
        assert b"lr_ratio" in lib.ngp_last_error()
    assert lib.ngp_pose_adam(None, None, None, None, None, None, 0.1, 0.9, 0.999, 1e-15, 0, None) == 0
    # the device-counted input gradient: every width, the usual checks
    bwd_x = lib.ngp_hash_encode_bwd_input_dyn
    for F in (1, 2, 4, 8):
        lay = make_hash_layout(2 ** 16, 6, 16, 512, F).as_ctypes()
        assert bwd_x(None, None, None, F32, C.byref(lay), None, 0, None, None, None) == 0
        assert bwd_x(fake, fake, fake, 7, C.byref(lay), fake, 8, None, None, None) < 0
        assert b"dtype" in lib.ngp_last_error()
        assert bwd_x(fake, None, fake, F32, C.byref(lay), fake, 8, None, None, None) < 0
        assert bwd_x(fake, fake, fake, F32, C.byref(lay), fake, -1, None, None, None) < 0
    bad = make_hash_layout(2 ** 16, 6, 16, 512, 2).as_ctypes()
    bad.feat_dim = 9
    assert bwd_x(fake, fake, fake, F32, C.byref(bad), fake, 8, None, None, None) < 0
    assert b"feature_per_level" in lib.ngp_last_error()


def test_refinement_state_refuses_bad_ratios():
    import torch
    from taichi_nerfs_b200.extrinsics import PoseRefinement
    for r in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="lr_ratio"):
            PoseRefinement(torch.zeros(2, 3, 4), r)
    with pytest.raises(ValueError, match="CUDA"):
        PoseRefinement(torch.zeros(2, 3, 4), 0.1)
