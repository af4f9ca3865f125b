"""Per-image exposure compensation (--exposure_lr, DESIGN.md §6k) without a GPU: the option's refusals, the fp64
restatement of apply, backward and Adam with the zero-mean projection on hand-computed cases, the C-ABI argument checks
of the three entries, and the kernels' register use (no spills) for sm_90a."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import exposure_ref as ref


# ---- opt.py ---------------------------------------------------------------------------------------------------------
def _opts(*args):
    from opt import get_opts
    return get_opts(list(args))


def test_exposure_lr_default_is_off():
    assert _opts().exposure_lr == 0.0
    assert _opts('--exposure_lr', '1e-3').exposure_lr == 1e-3


@pytest.mark.parametrize("v", ["-1e-3", "nan", "inf", "-inf"])
def test_exposure_lr_must_be_finite_and_non_negative(v, capsys):
    with pytest.raises(SystemExit):
        _opts(f'--exposure_lr={v}')
    assert "--exposure_lr must be finite and >= 0" in capsys.readouterr().err


@pytest.mark.parametrize("lr", ["0", "-1e-2", "nan", "inf"])
def test_exposure_lr_needs_a_positive_model_lr(lr, capsys):
    with pytest.raises(SystemExit):
        _opts('--exposure_lr', '1e-3', f'--lr={lr}')
    assert "needs a finite --lr > 0" in capsys.readouterr().err
    _opts('--exposure_lr', '0', f'--lr={lr}')   # off: --lr is not read by it


def test_exposure_lr_needs_one_rank(monkeypatch, capsys):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit):
        _opts('--exposure_lr', '1e-3')
    assert "one GPU" in capsys.readouterr().err
    _opts('--exposure_lr', '0')


@pytest.mark.parametrize("flags", [(), ('--model_name', 'svox'), ('--encoder_type', 'triplane'), ('--deployment',),
                                   ('--half_opt', '--graph_step')])
def test_exposure_lr_combines_with_every_model_kind(flags):
    assert _opts('--exposure_lr', '1e-3', *flags).exposure_lr == 1e-3


# ---- the restatement on hand-computed cases ---------------------------------------------------------------------------
def test_apply_scales_by_powers_of_two():
    rgbs = np.array([[0.5, 0.25, 1.0], [0.1, 0.2, 0.3], [0.7, 0.7, 0.7], [0.9, 0.9, 0.9]])
    rays_a = np.array([[0, 0, 2], [1, 2, 1], [2, 3, 0]])
    expo = np.array([[1.0, -1.0, 0.0, 0.0], [2.0, 0.5, -2.0, 0.0]])
    out = ref.apply(rgbs, rays_a, [1, 0, 0], expo)
    assert np.array_equal(out[0], [2.0, 0.25 * 2 ** 0.5, 0.25])
    assert np.array_equal(out[1], [0.4, 0.2 * 2 ** 0.5, 0.075])
    assert np.array_equal(out[2], [1.4, 0.35, 0.7])
    assert np.isnan(out[3]).all()   # a row of no ray
    # one index for the whole batch, and out-of-range indices clamped
    assert np.array_equal(ref.apply(rgbs, rays_a, [0], expo)[:3], ref.apply(rgbs, rays_a, [0, 0, 0], expo)[:3])
    assert np.array_equal(ref.apply(rgbs, rays_a, [7, -3, 5], expo)[:3], ref.apply(rgbs, rays_a, [1, 0, 1], expo)[:3])
    # e = 0 is the identity
    assert np.array_equal(ref.apply(rgbs, rays_a, [0, 1, 0], np.zeros((2, 4)))[:3], rgbs[:3])


def test_backward_by_hand():
    out = np.array([[2.0, 1.0, 0.5], [1.0, 1.0, 1.0], [0.5, 0.5, 0.5]])
    d = np.array([[1.0, 2.0, -1.0], [0.5, 0.5, 0.5], [4.0, 0.0, -4.0]])
    rays_a = np.array([[0, 0, 2], [1, 2, 1]])
    expo = np.array([[1.0, 0.0, -1.0, 0.0], [0.0, 0.0, 0.0, 0.0]])
    dc, grad, mag = ref.bwd(out, d, rays_a, [0, 1], expo)
    assert np.array_equal(dc[0], [2.0, 2.0, -0.5]) and np.array_equal(dc[1], [1.0, 0.5, 0.25])
    assert np.array_equal(dc[2], d[2])   # e = 0
    assert np.allclose(grad[0], np.log(2) * np.array([2.0 + 0.5, 2.0 + 0.5, -0.5 + 0.5]), rtol=0, atol=1e-15)
    assert np.allclose(grad[1], np.log(2) * np.array([2.0, 0.0, -2.0]), rtol=0, atol=1e-15)
    assert np.allclose(mag[0], np.log(2) * np.array([2.5, 2.5, 1.0]), rtol=0, atol=1e-15)


def test_backward_is_the_derivative_of_apply():
    """d/de of sum_s d_s . (2^e c_s) by central differences, at random exposures."""
    rng = np.random.default_rng(1)
    c = rng.random((40, 3))
    d = rng.standard_normal((40, 3))
    rays_a = np.array([[0, 0, 15], [1, 15, 10], [2, 25, 15]])
    img = np.array([1, 0, 1])
    e = np.c_[rng.uniform(-2, 2, (2, 3)), np.zeros(2)]
    _, grad, _ = ref.bwd(ref.apply(c, rays_a, img, e), d, rays_a, img, e)
    h = 1e-6
    for i in range(2):
        for ch in range(3):
            ep, em = e.copy(), e.copy()
            ep[i, ch] += h
            em[i, ch] -= h
            num = ((d * ref.apply(c, rays_a, img, ep)).sum() - (d * ref.apply(c, rays_a, img, em)).sum()) / (2 * h)
            assert abs(num - grad[i, ch]) < 1e-7 * max(1.0, abs(num))


def test_adam_first_step_and_projection_by_hand():
    """First step with bias correction (lr/bc1 = lr / (1 - b1), sqrt(bc2) = sqrt(1 - b2)): each exposure moves by
    lr_ratio lr sign(g) (eps = 0), then the per-channel mean is removed."""
    b1, b2, lr, ratio = 0.9, 0.999, 1e-2, 0.5
    hyper = (lr / (1 - b1), np.sqrt(1 - b2), 0.25)
    e0 = np.zeros((3, 3))
    g = np.array([[4.0, -8.0, 1.0], [-4.0, -8.0, 2.0], [2.0, 8.0, 3.0]])
    e, gz, m, v = ref.adam(e0, g, np.zeros((3, 3)), np.zeros((3, 3)), hyper, ratio, b1, b2, eps=0.0)
    step = -ratio * lr * np.sign(g)
    assert np.allclose(e, step - step.mean(0), rtol=0, atol=1e-17)
    assert np.allclose(m, (1 - b1) * g * 0.25) and np.allclose(v, (1 - b2) * (g * 0.25) ** 2)
    assert not gz.any()
    assert np.allclose(e.mean(0), 0, rtol=0, atol=1e-18)


def test_adam_skips_on_found_inf():
    e, g, m, v = np.ones((2, 3)), np.full((2, 3), np.inf), np.full((2, 3), 0.5), np.full((2, 3), 0.25)
    e1, g1, m1, v1 = ref.adam(e, g, m, v, (1.0, 1.0, 1.0), 0.1, found_inf=True)
    assert np.array_equal(e1, e) and np.array_equal(m1, m) and np.array_equal(v1, v) and not g1.any()


def test_adam_at_zero_rate_keeps_zero_exposures_exactly():
    g = np.random.default_rng(2).standard_normal((5, 3))
    e, _, _, _ = ref.adam(np.zeros((5, 3)), g, np.zeros((5, 3)), np.zeros((5, 3)), (0.1, 0.03, 1.0), 0.0)
    assert np.array_equal(e, np.zeros((5, 3)))


# ---- C-ABI argument checks (no launch) ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from taichi_nerfs_b200 import _lib, build
    build.build()
    return _lib.load()


def test_exposure_argument_validation_needs_no_gpu(lib):
    from taichi_nerfs_b200._lib import F16, F32
    fake, fake2, odd = C.c_void_p(0x10000), C.c_void_p(0x20000), C.c_void_p(0x10004)
    ap, bw, ad = lib.ngp_exposure_apply, lib.ngp_exposure_bwd, lib.ngp_exposure_adam
    # apply: negative counts, no images, bad dtype, null pointers, misaligned exposures, aliasing; n = 0 is a no-op
    assert ap(fake, F16, fake, fake, fake, 4, fake2, -1, 8, None, None) < 0
    assert ap(fake, F16, fake, fake, fake, 4, fake2, 8, -1, None, None) < 0
    assert ap(fake, F16, fake, fake, fake, 0, fake2, 8, 8, None, None) < 0
    assert b"n_img" in lib.ngp_last_error()
    assert ap(fake, 7, fake, fake, fake, 4, fake2, 8, 8, None, None) < 0
    assert b"dtype" in lib.ngp_last_error()
    assert ap(fake, F32, None, fake, fake, 4, fake2, 8, 8, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert ap(None, F32, fake, fake, fake, 4, None, 8, 8, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert ap(fake, F32, fake, fake, odd, 4, fake2, 8, 8, None, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert ap(fake, F32, fake, fake, fake, 4, fake, 8, 8, None, None) < 0
    assert b"alias" in lib.ngp_last_error()
    assert ap(None, F32, None, None, None, 4, None, 0, 0, None, None) == 0
    # backward
    assert bw(fake, fake2, F16, fake, fake, fake, 4, fake, None, -1, 8, None, None) < 0
    assert bw(fake, fake2, F16, fake, fake, fake, 0, fake, None, 8, 8, None, None) < 0
    assert bw(fake, fake2, 3, fake, fake, fake, 4, fake, None, 8, 8, None, None) < 0
    assert b"dtype" in lib.ngp_last_error()
    assert bw(fake, fake2, F16, fake, fake, fake, 4, None, None, 8, 8, None, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert bw(None, None, F16, fake, fake, fake, 4, fake, None, 8, 8, None, None) < 0
    assert bw(fake, fake2, F16, fake, fake, odd, 4, fake, None, 8, 8, None, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    assert bw(None, None, F16, None, None, None, 4, None, None, 0, 0, None, None) == 0
    # Adam
    assert ad(fake, fake, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, -1, None) < 0
    assert ad(fake, fake, fake, fake, None, None, 0.1, 0.9, 0.999, 1e-15, 4, None) < 0
    assert b"null" in lib.ngp_last_error()
    assert ad(fake, odd, fake, fake, None, fake, 0.1, 0.9, 0.999, 1e-15, 4, None) < 0
    assert b"aligned" in lib.ngp_last_error()
    for r in (-0.1, float("inf"), float("nan")):
        assert ad(fake, fake, fake, fake, None, fake, r, 0.9, 0.999, 1e-15, 4, None) < 0
        assert b"lr_ratio" in lib.ngp_last_error()
    assert ad(None, None, None, None, None, None, 0.1, 0.9, 0.999, 1e-15, 0, None) == 0


def test_correction_state_refuses_bad_arguments():
    from taichi_nerfs_b200.exposure import ExposureCorrection
    for r in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="lr_ratio"):
            ExposureCorrection(4, r, "cuda")
    with pytest.raises(ValueError, match="n_img"):
        ExposureCorrection(0, 0.1, "cuda")
    with pytest.raises(ValueError, match="CUDA"):
        ExposureCorrection(4, 0.1, "cpu")


# ---- registers and spills -------------------------------------------------------------------------------------------
def test_kernels_compile_for_sm90a_without_spills(tmp_path):
    from taichi_nerfs_b200 import build
    src = os.path.join(build.CSRC, "exposure.cu")
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "exposure.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True)
    log = out.stdout + out.stderr
    entries = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'", log)
    names = ("exposure_apply_kernel", "exposure_bwd_kernel", "exposure_adam_kernel")
    for k in names:
        assert any(k in e for e in entries), (k, log)
    assert len(entries) == 5, log   # apply and backward in fp32 and fp16, one Adam
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 5 and all(s == ("0", "0") for s in spills), log
    assert "bytes stack frame" in log and all(int(v) == 0 for v in re.findall(r"(\d+) bytes stack frame", log)), log
