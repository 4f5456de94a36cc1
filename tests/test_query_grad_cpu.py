"""Gradients of field queries without a GPU: workspace sizing of mipnerf_b200_query_backward, its binding, every
argument it refuses before it launches anything, and the refusals of the autograd path of MipNerf.query_density /
query_radiance (raised at query time, before any device work)."""
import ctypes as C

import pytest
import torch

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

FAKE = 256  # a non-NULL "device" pointer that no call below dereferences


def fake_weights(model):
    lins = model.mlp.linears()
    arr = (_cabi.Linear * len(lins))()
    for i, l in enumerate(lins):
        arr[i] = _cabi.Linear(FAKE, FAKE, l.in_features, l.out_features)
    return _cabi.Weights(arr, len(lins), -1, None, 0), arr


def fake_grads(model):
    n = len(model.mlp.linears())
    arr = (_cabi.LinearGrad * n)()
    for i in range(n):
        arr[i] = _cabi.LinearGrad(FAKE, FAKE)
    return arr


def backward(cfg, ws, grads, means=FAKE, covs=None, dirs=FAKE, p=8, precision=_cabi.FP32, cot=True, num_grads=None,
             work=FAKE, nbytes=1 << 40):
    c = _cabi.QueryCotangent(FAKE, FAKE, None, None)
    return _cabi.lib().mipnerf_b200_query_backward(
        C.byref(cfg) if cfg is not None else None, C.byref(ws), means, covs, dirs, p, precision,
        C.byref(c) if cot else None, grads, len(grads) if num_grads is None else num_grads, 0, work, nbytes, None)


def size(model, p, radiance, precision):
    return _cabi.lib().mipnerf_b200_query_backward_workspace_bytes(C.byref(model._config()), p, radiance, precision)


def test_symbols_are_bound():
    assert "mipnerf_b200_query_backward" in _cabi.EXPORTED_SYMBOLS
    assert "mipnerf_b200_query_backward_workspace_bytes" in _cabi.EXPORTED_SYMBOLS
    lib = _cabi.lib()
    assert lib.mipnerf_b200_query_backward.restype is C.c_int
    assert lib.mipnerf_b200_query_backward_workspace_bytes.restype is C.c_size_t
    assert [f for f, _ in _cabi.QueryCotangent._fields_] == ["d_raw_rgb", "d_raw_density", "d_rgb", "d_density"]


def test_workspace_sizing():
    model = mp.MipNerf()
    for radiance in (0, 1):
        for prec in (_cabi.FP32, _cabi.BF16):
            one, small, chunk = size(model, 1, radiance, prec), size(model, 1000, radiance, prec), size(
                model, 1 << 19, radiance, prec)
            assert 0 < one < small < chunk
            assert size(model, 1 << 26, radiance, prec) == chunk  # capped at one 524288-point chunk
            assert size(model, -1, radiance, prec) == 0
        for prec in (_cabi.FP16, _cabi.FP16X3, _cabi.BF16X3, 7):
            assert size(model, 1000, radiance, prec) == 0
    # a density query keeps no view-layer or colour-head activations
    assert size(model, 1000, 0, _cabi.FP32) < size(model, 1000, 1, _cabi.FP32)
    # configs the training chain refuses; BF16 with other encodings
    for kw in (dict(use_viewdirs=False, mlp_net_width_condition=256), dict(mlp_net_depth_condition=2),
               dict(mlp_net_depth=17)):
        assert size(mp.MipNerf(**kw), 1000, 1, _cabi.FP32) == 0
    for kw in (dict(max_deg_point=10), dict(deg_view=2), dict(mlp_net_depth=6)):
        other = mp.MipNerf(**kw)
        assert size(other, 1000, 1, _cabi.FP32) > 0
        assert size(other, 1000, 1, _cabi.BF16) == 0


def test_backward_refusals():
    model = mp.MipNerf()
    cfg = model._config()
    ws, _keep = fake_weights(model)
    grads = fake_grads(model)
    assert backward(None, ws, grads) == _cabi.EINVAL
    assert backward(cfg, ws, grads, p=-1) == _cabi.EINVAL
    assert backward(cfg, ws, grads, cot=False) == _cabi.EINVAL
    assert backward(cfg, ws, grads, num_grads=len(grads) - 1) == _cabi.EINVAL
    holes = fake_grads(model)
    holes[3] = _cabi.LinearGrad(FAKE, None)
    assert backward(cfg, ws, holes) == _cabi.EINVAL
    assert backward(cfg, ws, grads, means=None) == _cabi.EINVAL
    assert backward(cfg, ws, grads, precision=7) == _cabi.EINVAL
    assert backward(cfg, fake_weights(mp.MipNerf(max_deg_point=10))[0], grads) == _cabi.EINVAL  # weights of another shape
    for prec in (_cabi.FP16, _cabi.FP16X3, _cabi.BF16X3):
        assert backward(cfg, ws, grads, precision=prec) == _cabi.EUNSUPPORTED
    other = mp.MipNerf(deg_view=2)
    assert backward(other._config(), fake_weights(other)[0], fake_grads(other), precision=_cabi.BF16) == \
        _cabi.EUNSUPPORTED
    deep = mp.MipNerf(mlp_net_depth_condition=2)
    assert backward(deep._config(), fake_weights(deep)[0], fake_grads(deep)) == _cabi.EUNSUPPORTED
    need = size(model, 8, 1, _cabi.FP32)
    assert backward(cfg, ws, grads, nbytes=need - 1) == _cabi.EWORKSPACE
    assert backward(cfg, ws, grads, work=None) == _cabi.EWORKSPACE
    # a density query (viewdirs NULL) sizes its own, smaller workspace: past every argument check
    assert backward(cfg, ws, grads, dirs=None, nbytes=size(model, 8, 0, _cabi.FP32) - 1) == _cabi.EWORKSPACE
    assert backward(cfg, ws, grads, dirs=None, precision=_cabi.BF16, work=None) == _cabi.EWORKSPACE


def _autograd_model(**kw):
    return mp.MipNerf(autograd=True, **kw)


@pytest.mark.parametrize("precision", ["fp16", "fp16x3", "bf16x3"])
def test_python_refuses_precisions(precision):
    model = _autograd_model(precision=precision)
    x = torch.zeros(4, 3)
    with pytest.raises(NotImplementedError):
        model.query_density(x)
    with pytest.raises(NotImplementedError):
        model.query_radiance(x, None, x)


def test_python_refuses_configs_and_input_grads():
    x = torch.zeros(4, 3)
    for model in (_autograd_model(precision="bf16", max_deg_point=10), _autograd_model(mlp_net_depth_condition=2)):
        with pytest.raises(NotImplementedError):
            model.query_density(x)
        with pytest.raises(NotImplementedError):
            model.query_radiance(x, None, x)
    model = _autograd_model()
    for args in ((x.clone().requires_grad_(True), None, x), (x, x.clone().requires_grad_(True), x),
                 (x, None, x.clone().requires_grad_(True))):
        with pytest.raises(NotImplementedError):
            model.query_radiance(*args)
    with pytest.raises(NotImplementedError):
        model.query_density(x.clone().requires_grad_(True))
