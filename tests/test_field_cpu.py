"""Density queries and meshes without a GPU: the oracle's density against the reference's (tests/golden/field.npz), the
isosurface rules (tests/isosurface_ref.py) on analytic and random grids, PLY round trips, and every argument the C ABI
refuses before it launches anything."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import golden, make_state_dict, oracle
import isosurface_ref as R

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

CASES = ("xavier", "trained_like", "deg10_view2")


def oracle_raw_density(sd, means, covs, max_deg, view_dim=27):
    """oracle.integrated_pos_enc + trunk + density layer (the colour branch gets a zero view input it does not use)."""
    enc = oracle.integrated_pos_enc(means, covs, 0, max_deg)
    return oracle.mlp_forward(sd, enc[None], torch.zeros(1, view_dim))[1][0, :, 0]


@pytest.mark.parametrize("tag", CASES)
@pytest.mark.parametrize("cov", ["zero", "iso", "aniso"])
def test_oracle_density_matches_reference_golden(tag, cov):
    g = golden("field.npz")
    seed, max_deg, deg_view = (int(v) for v in g[f"{tag}_meta"])
    kind = "xavier" if tag == "xavier" else "trained_like"
    sd = make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3)
    got = oracle_raw_density(sd, torch.from_numpy(g[f"{tag}_means"]), torch.from_numpy(g[f"{tag}_covs_{cov}"]), max_deg,
                             6 * deg_view + 3)
    want = g[f"{tag}_raw_{cov}"]
    err = np.abs(got.numpy().astype(np.float64) - want) / np.maximum(np.abs(want), 1.0)
    assert err.max() <= 1e-5, err.max()


# ---- isosurface rules -------------------------------------------------------------------------------------------
def test_sphere_volume_and_topology():
    v, f, _ = R.isosurface(R.sphere_grid(64, 0.7), 0.0, ((-1.0,) * 3, (1.0,) * 3))
    vol = R.enclosed_volume(v, f)
    assert abs(vol - 4 / 3 * np.pi * 0.7 ** 3) <= 0.01 * 4 / 3 * np.pi * 0.7 ** 3, vol
    assert R.manifold_violations(f) == []
    assert R.euler_characteristic(v, f) == 2


def test_torus_topology():
    v, f, _ = R.isosurface(R.torus_grid(64, 0.55, 0.25), 0.0, ((-1.0,) * 3, (1.0,) * 3))
    assert R.manifold_violations(f) == []
    assert R.euler_characteristic(v, f) == 0
    assert R.enclosed_volume(v, f) > 0  # normals point out of the inside region


def test_random_grid_is_manifold_away_from_the_box():
    rng = np.random.RandomState(3)
    grid = rng.randn(11, 13, 17).astype(np.float32)
    grid[4, 5, 6] = np.nan  # NaN is outside
    v, f, e = R.isosurface(grid, 0.1, ((0.0, 0.0, 0.0), (1.0, 2.0, 3.0)))
    assert len(f) > 0 and np.isfinite(v).all()
    assert R.manifold_violations(f, R.on_box_face(e, (17, 13, 11))) == []
    assert R.manifold_violations(f) != []  # the open mesh does end on the box


def test_ply_round_trip(tmp_path):
    rng = np.random.RandomState(0)
    verts = rng.randn(37, 3).astype(np.float32)
    faces = rng.randint(0, 37, size=(50, 3)).astype(np.int32)
    path = os.path.join(tmp_path, "m.ply")
    mp.write_ply(path, torch.from_numpy(verts), torch.from_numpy(faces))
    with open(path, "rb") as fh:
        assert fh.read(3) == b"ply"
    v2, f2 = R.read_ply(path)
    assert np.array_equal(v2, verts) and np.array_equal(f2, faces)
    mp.write_ply(path, torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int32))
    v3, f3 = R.read_ply(path)
    assert v3.shape == (0, 3) and f3.shape == (0, 3)


# ---- host argument checks (nothing reaches a kernel) ---------------------------------------------------------------
FAKE = 256  # a non-NULL "device" pointer that no call below dereferences


def fake_weights(model, precision=-1, packed=0):
    lins = model.mlp.linears()
    arr = (_cabi.Linear * len(lins))()
    for i, l in enumerate(lins):
        arr[i] = _cabi.Linear(FAKE, FAKE, l.in_features, l.out_features)
    ws = _cabi.Weights(arr, len(lins), precision, packed or None, packed and (1 << 30))
    return ws, arr


def query(cfg, ws, means=FAKE, covs=None, p=8, precision=_cabi.FP32, raw=FAKE, dens=None, work=FAKE, nbytes=1 << 40):
    return _cabi.lib().mipnerf_b200_query_density(C.byref(cfg) if cfg is not None else None, C.byref(ws), means, covs,
                                                  p, precision, raw, dens, work, nbytes, None)


def test_query_density_refusals():
    lib = _cabi.lib()
    model = mp.MipNerf()
    cfg = model._config()
    ws, _keep = fake_weights(model)
    assert query(None, ws) == _cabi.EINVAL
    assert query(cfg, ws, p=-1) == _cabi.EINVAL
    assert query(cfg, ws, raw=None, dens=None) == _cabi.EINVAL
    assert query(cfg, ws, means=None) == _cabi.EINVAL
    assert query(cfg, ws, precision=7) == _cabi.EINVAL
    need = lib.mipnerf_b200_density_workspace_bytes(C.byref(cfg), 8, _cabi.FP32)
    assert need > 0
    assert query(cfg, ws, nbytes=need - 1) == _cabi.EWORKSPACE
    assert query(cfg, ws, work=None) == _cabi.EWORKSPACE
    # a workspace bounded by one launch chunk
    assert lib.mipnerf_b200_density_workspace_bytes(C.byref(cfg), 1 << 30, _cabi.FP32) == \
        lib.mipnerf_b200_density_workspace_bytes(C.byref(cfg), 1 << 20, _cabi.FP32)
    assert lib.mipnerf_b200_density_workspace_bytes(C.byref(cfg), -1, _cabi.FP32) == 0
    # tensor cores: the packed image must be there, for that precision; the forward's shapes only
    assert query(cfg, ws, precision=_cabi.BF16) == _cabi.EINVAL
    ws_bf, _k2 = fake_weights(model, _cabi.FP16, FAKE)
    assert query(cfg, ws_bf, precision=_cabi.BF16) == _cabi.EINVAL
    small = mp.MipNerf(num_samples=64)
    ws64, _k3 = fake_weights(small, _cabi.BF16, FAKE)
    assert query(small._config(), ws64, precision=_cabi.BF16) == _cabi.EUNSUPPORTED
    wrong = mp.MipNerf(max_deg_point=10)
    assert query(cfg, fake_weights(wrong)[0]) == _cabi.EINVAL   # weights of another shape
    # a 64-sample model still queries in fp32
    assert lib.mipnerf_b200_density_workspace_bytes(C.byref(small._config()), 8, _cabi.FP32) > 0


def test_isosurface_refusals():
    lib = _cabi.lib()
    assert lib.mipnerf_b200_isosurface_scratch_bytes(1, 2, 2) == 0
    need = lib.mipnerf_b200_isosurface_scratch_bytes(4, 3, 2)
    assert need > 0
    lo = (C.c_float * 3)(0, 0, 0)
    hi = (C.c_float * 3)(1, 1, 1)
    cnt = lib.mipnerf_b200_isosurface_count
    emit = lib.mipnerf_b200_isosurface_emit
    assert cnt(FAKE, 4, 3, 1, 0.0, FAKE, need, FAKE, None) == _cabi.EINVAL
    assert cnt(FAKE, -4, 3, 2, 0.0, FAKE, need, FAKE, None) == _cabi.EINVAL
    assert cnt(None, 4, 3, 2, 0.0, FAKE, need, FAKE, None) == _cabi.EINVAL
    assert cnt(FAKE, 4, 3, 2, 0.0, FAKE, need, None, None) == _cabi.EINVAL
    assert cnt(FAKE, 4, 3, 2, 0.0, FAKE, need - 1, FAKE, None) == _cabi.EWORKSPACE
    assert cnt(FAKE, 4, 3, 2, 0.0, None, need, FAKE, None) == _cabi.EWORKSPACE
    assert emit(FAKE, 4, 1, 2, lo, hi, 0.0, FAKE, FAKE, FAKE, None) == _cabi.EINVAL
    assert emit(None, 4, 3, 2, lo, hi, 0.0, FAKE, FAKE, FAKE, None) == _cabi.EINVAL
    assert emit(FAKE, 4, 3, 2, None, hi, 0.0, FAKE, FAKE, FAKE, None) == _cabi.EINVAL
    assert emit(FAKE, 4, 3, 2, lo, hi, 0.0, None, FAKE, FAKE, None) == _cabi.EINVAL
