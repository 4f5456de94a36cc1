"""MipNerf(autograd=True) without a GPU: the C-ABI structs, the module surface and the CPU-tensor refusal."""
import ctypes as C

import pytest
import torch

import helpers  # noqa: F401  (puts the repository root on sys.path)
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi


def test_level_cotangent_struct_matches_header():
    assert C.sizeof(_cabi.LevelCotangent) == 4 * 8
    assert [f for f, _ in _cabi.LevelCotangent._fields_] == ["d_comp_rgb", "d_distance", "d_acc", "d_weights"]
    assert {"mipnerf_b200_backward", "mipnerf_b200_distloss_backward"} <= set(_cabi.EXPORTED_SYMBOLS)


def test_autograd_flag_keeps_the_module_surface():
    plain, grad = mp.MipNerf(), mp.MipNerf(autograd=True)
    assert not plain.autograd and grad.autograd
    assert list(plain.state_dict()) == list(grad.state_dict())
    assert [n for n, _ in plain.named_parameters()] == [n for n, _ in grad.named_parameters()]
    grad.load_state_dict(plain.state_dict())


def test_autograd_forward_on_cpu_tensors_raises():
    model = mp.MipNerf(autograd=True)
    rays = mp.random_ray_batch(8, seed=1, multiscale=True)
    assert torch.is_grad_enabled() and all(p.requires_grad for p in model.parameters())
    with pytest.raises(RuntimeError):
        model(rays, False, True)


def test_bf16_autograd_refuses_at_forward_time_what_the_backward_refuses():
    """Depth 16 with skip index 2 has the default widths, but the per-layer tensor-core step cannot hold its weight
    images, so the bf16 backward would refuse it: the forward's precondition asks the library and refuses it first."""
    from mipnerf_pl_b200 import mip_nerf
    model = mp.MipNerf(mlp_net_depth=16, mlp_skip_index=2, precision="bf16", autograd=True)
    rays = mp.random_ray_batch(8, seed=1, multiscale=True)
    cfg = model._config()
    assert _cabi.lib().mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), 8, _cabi.FP32) > 0
    assert _cabi.lib().mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), 8, _cabi.BF16) == 0
    with pytest.raises(NotImplementedError, match="tensor-core backward"):
        mip_nerf._check_autograd(model, rays, 8)
