"""Workspace sizing of the training step per precision (no GPU needed): the precision-free entry point keeps what it
returned before the bf16x3 step existed, and bf16x3 has a size only where its fused step runs."""
import ctypes as C

import pytest

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


CONFIGS = {"default": {}, "one level": {"num_levels": 1}, "64 samples": {"num_samples": 64},
           "three levels": {"num_levels": 3}, "deg 10": {"max_deg_point": 10}, "depth 4": {"mlp_net_depth": 4},
           "no viewdirs": {"use_viewdirs": False, "mlp_net_width_condition": 256}}


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("rays", [0, 1, 37, 2048, 4096, 4096 + 37, 10 ** 6])
def test_train_workspace_is_the_max_over_the_non_split_precisions(lib, name, rays):
    cfg = mp.MipNerf(**CONFIGS[name])._config()
    per = [lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), rays, p) for p in (_cabi.FP32, _cabi.BF16, _cabi.FP16)]
    assert lib.mipnerf_b200_train_workspace_bytes(C.byref(cfg), rays) == max(per)
    x3 = lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), rays, _cabi.BF16X3)
    fused = name in ("default", "one level")  # 8x256 / 1x128, default encodings, 128 samples, <= 2 levels
    assert (x3 > 0) == fused, (name, x3)
    assert lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), rays, _cabi.FP16X3) == 0
    if fused and rays >= 2048:  # 2048-ray chunks: no larger than the 16-bit step's 4096-ray chunk
        assert x3 == lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), 2048, _cabi.BF16X3)
        assert x3 <= lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), 4096, _cabi.BF16)
