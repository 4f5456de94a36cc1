"""Refusals of the loop kernels' entry points (Adam, image metrics, the frame ray generator, the pixel ray bank) and of
DeviceRayBank, all of which happen before anything touches a device, so they run without a GPU."""
import ctypes as C

import numpy as np
import pytest

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

FAKE = 256  # a non-NULL "device" pointer that no call below dereferences


def lib():
    return _cabi.lib()


def adam_multi(count, params, grads, exp_avg, exp_avg_sq, sizes):
    return lib().mipnerf_b200_adam_step_multi(count, params, grads, exp_avg, exp_avg_sq, sizes, 1e-3, 0.9, 0.999, 1e-8,
                                              1, 1.0, None)


def test_adam_step_multi_refusals():
    n = 65
    ptrs = (C.c_void_p * n)(*([FAKE] * n))
    nulls = (C.c_void_p * n)()
    zeros = (C.c_int64 * n)()
    assert adam_multi(-1, None, None, None, None, None) == _cabi.EINVAL
    assert adam_multi(0, None, None, None, None, None) == _cabi.OK
    assert adam_multi(1, None, ptrs, ptrs, ptrs, zeros) == _cabi.EINVAL
    for k in range(5):   # each host array NULL in turn
        args = [ptrs, ptrs, ptrs, ptrs, zeros]
        args[k] = None
        assert adam_multi(3, *args) == _cabi.EINVAL, k
    assert adam_multi(n, nulls, nulls, nulls, nulls, zeros) == _cabi.OK   # zero-size tensors need no pointers
    # a negative size anywhere, in the first, second or third launch's 32 tensors, is refused before any launch
    for i in (0, 31, 32, 63, 64):
        sizes = (C.c_int64 * n)()
        sizes[i] = -1
        assert adam_multi(n, nulls, nulls, nulls, nulls, sizes) == _cabi.EINVAL, i
        assert f"tensor {i}".encode() in lib().mipnerf_b200_last_error()
    # a NULL pointer of a non-empty tensor after non-empty tensors with valid pointers: refused before their launch
    sizes = (C.c_int64 * n)(*([5] * n))
    for k in range(4):
        arrays = [ptrs, ptrs, ptrs, ptrs]
        arrays[k] = (C.c_void_p * n)(*([FAKE] * 40 + [0] * 25))
        assert adam_multi(n, *arrays, sizes) == _cabi.EINVAL, k
        assert b"tensor 40" in lib().mipnerf_b200_last_error()


def test_image_metrics_refusals():
    need = lib().mipnerf_b200_image_metrics_scratch_bytes(37, 29, 3)
    assert need == 2 * 8 * 2 * 3 * 3
    for h, w, c in ((0, 5, 3), (5, 0, 3), (5, 5, 0), (-1, 5, 3)):
        assert lib().mipnerf_b200_image_metrics_scratch_bytes(h, w, c) == 0
        assert lib().mipnerf_b200_image_metrics(FAKE, FAKE, h, w, c, FAKE, 1 << 20, FAKE, None) == _cabi.EINVAL
    for scratch, nbytes in ((FAKE, need - 1), (FAKE, 0), (None, need)):
        assert lib().mipnerf_b200_image_metrics(FAKE, FAKE, 37, 29, 3, scratch, nbytes, FAKE, None) == _cabi.EWORKSPACE
    for pred, target, out in ((None, FAKE, FAKE), (FAKE, None, FAKE), (FAKE, FAKE, None)):
        assert lib().mipnerf_b200_image_metrics(pred, target, 37, 29, 3, FAKE, need, out, None) == _cabi.EINVAL


def generate(height, width, focal, row0, rows, outputs=FAKE, pose=True):
    c2w = np.ascontiguousarray(mp.spheric_pose(0.3)).reshape(-1)
    p = c2w.ctypes.data_as(C.POINTER(C.c_float)) if pose else None
    return lib().mipnerf_b200_generate_rays(p, height, width, focal, 2.0, 6.0, row0, rows, *([outputs] * 6), None)


def test_generate_rays_refusals():
    for h, w, f, r0, rows in ((1, 5, 10.0, 0, 1), (0, 5, 10.0, 0, 0), (4, 0, 10.0, 0, 4), (4, 5, 0.0, 0, 4),
                              (4, 5, -1.0, 0, 4), (4, 5, float("nan"), 0, 4), (4, 5, 10.0, 0, 5), (4, 5, 10.0, 3, 2),
                              (4, 5, 10.0, -1, 2), (4, 5, 10.0, 0, -1), (4, 5, 10.0, 5, 0)):
        assert generate(h, w, f, r0, rows) == _cabi.EINVAL, (h, w, f, r0, rows)
    assert generate(4, 5, 10.0, 0, 4, pose=False) == _cabi.EINVAL
    assert generate(4, 5, 10.0, 1, 2, outputs=None) == _cabi.EINVAL
    for r0 in (0, 2, 4):   # an empty row range is accepted and launches nothing
        assert generate(4, 5, 10.0, r0, 0, outputs=None) == _cabi.OK


def test_rays_from_pixels_refusals():
    f = lib().mipnerf_b200_rays_from_pixels
    outs = [FAKE] * 7
    assert f(FAKE, FAKE, FAKE, 3, FAKE, 4, None, *outs, FAKE, None) == _cabi.EINVAL   # rgb without an atlas
    assert b"atlas" in lib().mipnerf_b200_last_error()
    assert f(FAKE, FAKE, FAKE, 3, None, 0, None, *outs, FAKE, None) == _cabi.EINVAL
    assert f(FAKE, FAKE, FAKE, 0, None, 0, None, *outs, None, None) == _cabi.EINVAL
    assert f(FAKE, FAKE, FAKE, 3, None, -1, None, *outs, None, None) == _cabi.EINVAL
    assert f(FAKE, FAKE, FAKE, 3, None, 4, None, *outs, None, None) == _cabi.EINVAL   # count > 0 needs the ids
    assert f(FAKE, FAKE, FAKE, 3, None, 0, None, *([None] * 7), None, None) == _cabi.OK


def test_device_ray_bank_refuses_scenes_without_pixels():
    """A scene with no pixels would send every id to atlas row -1; the constructor refuses it before it touches the
    device, as it does a scene with no images."""
    def scene(shapes):
        n = len(shapes)
        return mp.Scene([np.zeros(s + (3,), np.float32) for s in shapes], np.zeros((n, 3, 3)), np.zeros((n, 3, 4)),
                        1.0, 2.0, 6.0)
    with pytest.raises(ValueError, match="no images"):
        mp.DeviceRayBank(scene([]), "cuda")
    for shapes in ([(0, 5)], [(4, 0)], [(0, 0), (0, 7), (3, 0)]):
        with pytest.raises(ValueError, match="no pixels"):
            mp.DeviceRayBank(scene(shapes), "cuda")
    with pytest.raises(RuntimeError, match="HBM"):
        mp.DeviceRayBank(scene([(2, 2)]), "cpu")
