"""256 samples per level, without a GPU: the oracle against the reference's own 256-sample forwards
(tests/golden/forward_n256*.npz), and the tensor-core shape contract through the C ABI (the level kernel takes a ray of
256 samples as two 128-row tiles, with the same operand image as at 128)."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import assert_level_close, golden, golden_levels, golden_rays, make_state_dict, oracle, oracle_rays

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

TC_PRECISIONS = (_cabi.BF16, _cabi.FP16, _cabi.FP16X3, _cabi.BF16X3)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def bit_equal(a, b, what):
    a = a.numpy() if isinstance(a, torch.Tensor) else a
    assert a.shape == b.shape, what
    bad = np.flatnonzero(~((a == b) | (np.isnan(a) & np.isnan(b))))
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} elements differ, first at {bad[:5]}"


@pytest.mark.parametrize("name,cfg", [
    ("forward_n256.npz", dict(num_samples=256)),
    ("forward_n256_randomized.npz", dict(num_samples=256, density_noise=1.0)),
])
def test_oracle_matches_reference_at_256_samples(name, cfg):
    g = golden(name)
    seed, randomized, white = (int(v) for v in g["meta"])
    assert g["l0_t_samples"].shape[1] == 257 and g["l1_inds"].shape[1] == 257
    params = make_state_dict(seed=seed, kind="trained_like")
    rays = oracle_rays(golden_rays(g))
    t_rand = torch.from_numpy(g["t_rand"]) if "t_rand" in g else None
    u_jit = torch.from_numpy(g["u_jitter"]) if "u_jitter" in g else None
    normals = ([torch.from_numpy(g[f"density_normal_l{lvl}"]) for lvl in range(2)]
               if "density_normal_l0" in g else None)
    ret, dbg = oracle.forward(params, rays, bool(randomized), bool(white), cfg, t_rand=t_rand, u_jitter=u_jit,
                              return_debug=True, density_normal=normals)
    want = golden_levels(g)
    assert len(ret) == len(want) == 2
    for lvl, (got, ref) in enumerate(zip(ret, want)):
        assert_level_close(got, ref, what=f"{name} level {lvl} ", level=lvl)
        bit_equal(got[4], ref[4], f"{name} level {lvl} t_samples")
        if lvl > 0:
            bit_equal(dbg[lvl]["inds"], g[f"l{lvl}_inds"], f"{name} level {lvl} inds")
    bit_equal(ret[0][3], want[0][3], f"{name} coarse weights")


def test_tensor_core_shape_contract_at_256_samples(lib):
    n128 = mp.MipNerf()._config()
    n256 = mp.MipNerf(num_samples=256)._config()
    for prec in TC_PRECISIONS:
        packed = lib.mipnerf_b200_packed_weights_bytes(C.byref(n256), prec)
        assert packed > 0 and packed == lib.mipnerf_b200_packed_weights_bytes(C.byref(n128), prec), prec
        assert lib.mipnerf_b200_workspace_bytes(C.byref(n256), 4096, prec) > 0, prec
        assert lib.mipnerf_b200_workspace_bytes(C.byref(n256), 1, prec) > 0, prec
        # the workspace is bounded by the chunk of rays per launch
        assert lib.mipnerf_b200_workspace_bytes(C.byref(n256), 10 ** 7, prec) == \
            lib.mipnerf_b200_workspace_bytes(C.byref(n256), 10 ** 8, prec), prec
    # narrower encodings at 256 samples: the zero-padded image, as at 128
    narrow = mp.MipNerf(num_samples=256, max_deg_point=10, deg_view=2)._config()
    narrow128 = mp.MipNerf(max_deg_point=10, deg_view=2)._config()
    assert lib.mipnerf_b200_packed_weights_bytes(C.byref(narrow), _cabi.BF16) == \
        lib.mipnerf_b200_packed_weights_bytes(C.byref(narrow128), _cabi.BF16) > 0
    for n in (32, 64, 96, 192):
        other = mp.MipNerf(num_samples=n)._config()
        for prec in TC_PRECISIONS:
            assert lib.mipnerf_b200_packed_weights_bytes(C.byref(other), prec) == 0, (n, prec)
            assert lib.mipnerf_b200_workspace_bytes(C.byref(other), 16, prec) == 0, (n, prec)
        assert lib.mipnerf_b200_workspace_bytes(C.byref(other), 16, _cabi.FP32) > 0, n   # the fp32 path takes it


@pytest.mark.parametrize("n", [64, 192])
def test_tensor_core_refusal_names_both_sample_counts(lib, n):
    model = mp.MipNerf(num_samples=n, precision="bf16")
    with pytest.raises(NotImplementedError, match="num_samples 128 or 256"):
        model.mlp._packed_image(model._config(), None, _cabi.BF16, "cpu", [])
