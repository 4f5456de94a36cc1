"""The config space of tests/test_gpu_config_space.py without a GPU: the C ABI accepts every entry of its table (so the
table cannot drift into configs the library refuses), and refuses, before it launches anything, the two shapes it does
not train or render: a per-layer tensor-core step whose packed weight images overflow the workspace's 40 slots, and a
view-conditioned model without view layers."""
import ctypes as C

import pytest

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi
from test_gpu_config_space import CONFIGS, TABLE

FAKE = 256  # a non-NULL "device" pointer that no call below dereferences


def fake_weights(model):
    """Weights of the model's shapes (tests/test_radiance_dirs_cpu.py builds them the same way)."""
    lins = model.mlp.linears()
    arr = (_cabi.Linear * len(lins))()
    for i, l in enumerate(lins):
        arr[i] = _cabi.Linear(FAKE, FAKE, l.in_features, l.out_features)
    return _cabi.Weights(arr, len(lins), -1, None, 0), arr


def zero_ray_forward(model, precision=_cabi.FP32):
    cfg = model._config()
    ws, keep = fake_weights(model)
    rays = _cabi.RaysStruct(None, None, None, None, None, None, 0)
    outs = (_cabi.LevelOut * model.num_levels)()
    return _cabi.lib().mipnerf_b200_forward(C.byref(cfg), C.byref(ws), C.byref(rays), 0, None, None, 1, precision, outs,
                                            None, 0, None)


def zero_ray_training_step(model, precision):
    cfg = model._config()
    ws, keep = fake_weights(model)
    rays = _cabi.RaysStruct(None, None, None, None, None, None, 0)
    levels = model.num_levels
    mult = (C.c_float * levels)(*([1.0] * levels))
    loss = _cabi.Loss(None, None, None, 1.0, mult, mult, None, None)
    outs = (_cabi.LevelOut * levels)()
    n_lin = len(model.mlp.linears())
    grads = (_cabi.LinearGrad * n_lin)(*[_cabi.LinearGrad(FAKE, FAKE) for _ in range(n_lin)])
    # accumulate=1: with no rays there is then nothing to zero either, so nothing touches the fake pointers
    return _cabi.lib().mipnerf_b200_forward_backward(C.byref(cfg), C.byref(ws), C.byref(rays), 0, None, None, 1,
                                                     precision, C.byref(loss), outs, grads, n_lin, 1, None, 0, None)


@pytest.mark.parametrize("cid", list(CONFIGS))
def test_abi_accepts_every_table_entry(cid):
    assert set(TABLE) <= set(CONFIGS)
    model = mp.MipNerf(**CONFIGS[cid])
    cfg = model._config()
    lib = _cabi.lib()
    for rays in (1, 333, 4096 + 37):
        assert lib.mipnerf_b200_workspace_bytes(C.byref(cfg), rays, _cabi.FP32) > 0, _cabi.last_error()
    rc = zero_ray_forward(model)
    assert rc not in (_cabi.EINVAL, _cabi.EUNSUPPORTED), (rc, _cabi.last_error())
    assert rc == _cabi.OK


def test_tensor_core_step_refuses_more_weight_images_than_slots():
    """Depth 16 with skip index 2: 7 skip layers, 4 + 16 + 15 + 7 = 42 packed images > 40 slots.  The fp32 step takes
    it; the per-layer tensor-core step has no workspace size for it and refuses the call.  Depth 16 with skip index 4
    (38 images) is the deepest that fits."""
    lib = _cabi.lib()
    deep = mp.MipNerf(mlp_net_depth=16, mlp_skip_index=2, num_samples=32, num_levels=1)
    cfg = deep._config()
    assert lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), 100, _cabi.FP32) > 0
    for prec in (_cabi.BF16, _cabi.FP16):
        assert lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), 100, prec) == 0
        assert zero_ray_training_step(deep, prec) == _cabi.EUNSUPPORTED
    assert zero_ray_training_step(deep, _cabi.FP32) == _cabi.OK
    fits = mp.MipNerf(mlp_net_depth=16, mlp_skip_index=4, num_samples=32, num_levels=1)
    for prec in (_cabi.FP32, _cabi.BF16, _cabi.FP16):
        assert lib.mipnerf_b200_train_workspace_bytes_for(C.byref(fits._config()), 100, prec) > 0
        assert zero_ray_training_step(fits, prec) == _cabi.OK


def test_view_conditioned_model_without_view_layers_is_refused():
    """use_viewdirs with net_depth_condition=0: the colour head would read net_width + view_dim inputs, which the
    reference's color_layer (net_width_condition inputs) cannot take.  Refused by every entry point before anything
    runs: no workspace size, and a forward without rays already returns EUNSUPPORTED."""
    lib = _cabi.lib()
    model = mp.MipNerf(mlp_net_depth_condition=0)
    cfg = model._config()
    assert lib.mipnerf_b200_workspace_bytes(C.byref(cfg), 100, _cabi.FP32) == 0
    assert zero_ray_forward(model) == _cabi.EUNSUPPORTED
    assert zero_ray_training_step(model, _cabi.FP32) == _cabi.EUNSUPPORTED
    # without view conditioning the view layers are unused, and the model is fine
    plain = mp.MipNerf(mlp_net_depth_condition=0, use_viewdirs=False, mlp_net_width_condition=256)
    assert lib.mipnerf_b200_workspace_bytes(C.byref(plain._config()), 100, _cabi.FP32) > 0
    assert zero_ray_forward(plain) == _cabi.OK
