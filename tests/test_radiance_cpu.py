"""Radiance queries and coloured meshes without a GPU: the oracle's radiance against the reference's
(tests/golden/radiance.npz), the vertex-normal rule (tests/isosurface_normals_ref.py) on analytic grids, PLY files with
normals and colours, and every argument the new C ABI entry points refuse before they launch anything."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import golden, make_state_dict, oracle
import isosurface_ref as R
import isosurface_normals_ref as NR

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

CASES = ("xavier", "trained_like", "deg10_view2")


def oracle_radiance(sd, means, covs, dirs, max_deg, deg_view):
    """oracle.integrated_pos_enc + oracle.pos_enc + oracle.mlp_forward on [P,1,xyz_dim] with [P,view_dim]."""
    enc = oracle.integrated_pos_enc(means, covs, 0, max_deg)[:, None]
    venc = oracle.pos_enc(dirs, 0, deg_view, True)
    raw_rgb, raw_density = oracle.mlp_forward(sd, enc, venc)
    return raw_rgb[:, 0], raw_density[:, 0, 0]


@pytest.mark.parametrize("tag", CASES)
@pytest.mark.parametrize("cov", ["zero", "iso", "aniso"])
def test_oracle_radiance_matches_reference_golden(tag, cov):
    g = golden("radiance.npz")
    seed, max_deg, deg_view = (int(v) for v in g[f"{tag}_meta"])
    kind = "xavier" if tag == "xavier" else "trained_like"
    sd = make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3)
    rgb, dens = oracle_radiance(sd, torch.from_numpy(g[f"{tag}_means"]), torch.from_numpy(g[f"{tag}_covs_{cov}"]),
                                torch.from_numpy(g[f"{tag}_viewdirs"]), max_deg, deg_view)
    for got, want in ((rgb, g[f"{tag}_raw_rgb_{cov}"]), (dens, g[f"{tag}_raw_density_{cov}"])):
        err = np.abs(got.numpy().astype(np.float64) - want) / np.maximum(np.abs(want), 1.0)
        assert err.max() <= 1e-5, err.max()


def test_golden_shares_field_points():
    """radiance.npz is taken at field.npz's points, so the two goldens agree on the raw density."""
    f, r = golden("field.npz"), golden("radiance.npz")
    for tag in CASES:
        assert np.array_equal(f[f"{tag}_means"], r[f"{tag}_means"])
        for cov in ("zero", "iso", "aniso"):
            err = np.abs(f[f"{tag}_raw_{cov}"] - r[f"{tag}_raw_density_{cov}"]) / np.maximum(
                np.abs(f[f"{tag}_raw_{cov}"]), 1.0)
            assert err.max() <= 1e-5
        d = r[f"{tag}_viewdirs"]
        assert np.allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-6)


# ---- vertex normals ---------------------------------------------------------------------------------------------
def test_sphere_normals_are_radial():
    bounds = ((-1.0,) * 3, (1.0,) * 3)
    v, f, n = NR.normals(R.sphere_grid(64, 0.7), 0.0, bounds)
    assert n.dtype == np.float32 and n.shape == v.shape
    radial = v / np.linalg.norm(v, axis=1, keepdims=True)
    cos = (n.astype(np.float64) * radial).sum(axis=1)
    assert np.all(np.abs(np.linalg.norm(n, axis=1) - 1) < 1e-6)
    assert cos.min() > np.cos(np.radians(3.0)), np.degrees(np.arccos(cos.min()))


@pytest.mark.parametrize("name", ["sphere", "torus"])
def test_normals_agree_with_face_orientation(name):
    grid = R.sphere_grid(48, 0.6) if name == "sphere" else R.torus_grid(48, 0.55, 0.25)
    v, f, n = NR.normals(grid, 0.0, ((-1.0,) * 3, (1.0,) * 3))
    fn = NR.face_normals(v, f)
    assert np.all((n.astype(np.float64) * fn).sum(axis=1) > 0)


def test_normals_with_nan_and_box_faces():
    rng = np.random.RandomState(3)
    grid = rng.randn(11, 13, 17).astype(np.float32)
    grid[4, 5, 6] = np.nan
    v, f, n = NR.normals(grid, 0.1, ((0.0, 0.0, 0.0), (1.0, 2.0, 3.0)))
    length = np.linalg.norm(n, axis=1)
    zero = length == 0
    assert zero.any() and not zero.all()   # the NaN's neighbours have no normal, the others a unit one
    assert np.all(np.abs(length[~zero] - 1) < 1e-6) and np.isfinite(n).all()


def test_linear_field_normals_exact():
    """A linear field has the same gradient everywhere, at the box faces too: every normal is -grad / |grad|."""
    xs = np.linspace(0.0, 1.0, 9, dtype=np.float32)
    z, y, x = np.meshgrid(xs, xs, xs, indexing="ij")
    grid = (0.5 - x).astype(np.float32)   # inside: x < 0.5, so the outward normal is +x
    v, f, n = NR.normals(grid, 0.0, ((0.0,) * 3, (1.0,) * 3))
    assert len(v) > 0 and np.allclose(n, [1.0, 0.0, 0.0], atol=1e-6)


# ---- PLY --------------------------------------------------------------------------------------------------------
def read_ply_full(path):
    """(header lines, vertex record array, faces) of a binary PLY whose vertex properties are float or uchar."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    props = []
    for h in header[header.index(next(h for h in header if h.startswith("element vertex"))) + 1:]:
        if not h.startswith("property"):
            break
        _, typ, name = h.split()
        props.append((name, "<f4" if typ == "float" else "u1"))
    rec = np.frombuffer(data, dtype=props, count=nv, offset=end)
    off = end + rec.nbytes
    fr = np.frombuffer(data, dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=nf, offset=off)
    assert (fr["n"] == 3).all() and off + 13 * nf == len(data)
    return header, rec, fr["idx"].copy()


def test_ply_with_normals_and_colors_round_trips(tmp_path):
    rng = np.random.RandomState(0)
    verts = rng.randn(37, 3).astype(np.float32)
    faces = rng.randint(0, 37, size=(50, 3)).astype(np.int32)
    normals = rng.randn(37, 3).astype(np.float32)
    colors = rng.uniform(-0.2, 1.2, size=(37, 3)).astype(np.float32)
    path = os.path.join(tmp_path, "c.ply")
    mp.write_ply(path, torch.from_numpy(verts), torch.from_numpy(faces), colors=torch.from_numpy(colors),
                 normals=torch.from_numpy(normals))
    header, rec, f2 = read_ply_full(path)
    assert [h for h in header if h.startswith("property")][:9] == [
        "property float x", "property float y", "property float z", "property float nx", "property float ny",
        "property float nz", "property uchar red", "property uchar green", "property uchar blue"]
    assert np.array_equal(np.stack([rec["x"], rec["y"], rec["z"]], 1), verts)
    assert np.array_equal(np.stack([rec["nx"], rec["ny"], rec["nz"]], 1), normals)
    want = np.round(np.clip(colors, 0, 1) * 255).astype(np.uint8)
    assert np.array_equal(np.stack([rec["red"], rec["green"], rec["blue"]], 1), want)
    assert np.array_equal(f2, faces)
    # colours only
    mp.write_ply(path, verts, faces, colors=colors)
    header, rec, f3 = read_ply_full(path)
    assert rec.dtype.names == ("x", "y", "z", "red", "green", "blue") and np.array_equal(f3, faces)


def test_ply_without_extras_is_unchanged(tmp_path):
    """Without colours and normals the file is the plain x, y, z PLY byte for byte."""
    rng = np.random.RandomState(1)
    verts = rng.randn(11, 3).astype(np.float32)
    faces = rng.randint(0, 11, size=(7, 3)).astype(np.int32)
    path = os.path.join(tmp_path, "p.ply")
    mp.write_ply(path, verts, faces)
    rec = np.empty(len(faces), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    rec["n"], rec["idx"] = 3, faces
    want = (b"ply\nformat binary_little_endian 1.0\nelement vertex 11\nproperty float x\nproperty float y\n"
            b"property float z\nelement face 7\nproperty list uchar int vertex_indices\nend_header\n" +
            verts.astype("<f4").tobytes() + rec.tobytes())
    with open(path, "rb") as fh:
        assert fh.read() == want


# ---- host argument checks (nothing reaches a kernel) ---------------------------------------------------------------
FAKE = 256  # a non-NULL "device" pointer that no call below dereferences


def fake_weights(model, precision=-1, packed=0):
    lins = model.mlp.linears()
    arr = (_cabi.Linear * len(lins))()
    for i, l in enumerate(lins):
        arr[i] = _cabi.Linear(FAKE, FAKE, l.in_features, l.out_features)
    ws = _cabi.Weights(arr, len(lins), precision, packed or None, packed and (1 << 30))
    return ws, arr


def query(cfg, ws, means=FAKE, covs=None, dirs=FAKE, p=8, precision=_cabi.FP32, outs=(FAKE, None, None, None),
          work=FAKE, nbytes=1 << 40):
    return _cabi.lib().mipnerf_b200_query_radiance(C.byref(cfg) if cfg is not None else None, C.byref(ws), means,
                                                   covs, dirs, p, precision, *outs, work, nbytes, None)


def test_query_radiance_refusals():
    lib = _cabi.lib()
    model = mp.MipNerf()
    cfg = model._config()
    ws, _keep = fake_weights(model)
    assert query(None, ws) == _cabi.EINVAL
    assert query(cfg, ws, p=-1) == _cabi.EINVAL
    assert query(cfg, ws, outs=(None, None, None, None)) == _cabi.EINVAL
    assert query(cfg, ws, means=None) == _cabi.EINVAL
    assert query(cfg, ws, dirs=None) == _cabi.EINVAL
    assert query(cfg, ws, precision=7) == _cabi.EINVAL
    need = lib.mipnerf_b200_radiance_workspace_bytes(C.byref(cfg), 8, _cabi.FP32)
    assert need > 0
    assert query(cfg, ws, nbytes=need - 1) == _cabi.EWORKSPACE
    assert query(cfg, ws, work=None) == _cabi.EWORKSPACE
    assert lib.mipnerf_b200_radiance_workspace_bytes(C.byref(cfg), 1 << 30, _cabi.FP32) == \
        lib.mipnerf_b200_radiance_workspace_bytes(C.byref(cfg), 1 << 20, _cabi.FP32)
    assert lib.mipnerf_b200_radiance_workspace_bytes(C.byref(cfg), -1, _cabi.FP32) == 0
    # tensor cores: the packed image must be there, for that precision; the forward's shapes only
    assert query(cfg, ws, precision=_cabi.BF16) == _cabi.EINVAL
    ws_fp16, _k2 = fake_weights(model, _cabi.FP16, FAKE)
    assert query(cfg, ws_fp16, precision=_cabi.BF16) == _cabi.EINVAL
    small = mp.MipNerf(num_samples=64)
    ws64, _k3 = fake_weights(small, _cabi.BF16, FAKE)
    assert query(small._config(), ws64, precision=_cabi.BF16) == _cabi.EUNSUPPORTED
    assert lib.mipnerf_b200_radiance_workspace_bytes(C.byref(small._config()), 8, _cabi.BF16) == 0
    wrong = mp.MipNerf(max_deg_point=10)
    assert query(cfg, fake_weights(wrong)[0]) == _cabi.EINVAL   # weights of another shape
    # use_viewdirs=False: viewdirs may be NULL (fp32); the tensor cores refuse the config
    nov = mp.MipNerf(use_viewdirs=False, mlp_net_width_condition=256)
    ws_nov, _k4 = fake_weights(nov)
    assert query(nov._config(), ws_nov, dirs=None, work=None) == _cabi.EWORKSPACE  # past every argument check
    ws_nov_bf, _k5 = fake_weights(nov, _cabi.BF16, FAKE)
    assert query(nov._config(), ws_nov_bf, dirs=None, precision=_cabi.BF16) == _cabi.EUNSUPPORTED
    # use_viewdirs=False needs the reference's colour-layer shape
    bad = model._config()
    bad.use_viewdirs = 0
    assert query(bad, ws, dirs=None) == _cabi.EUNSUPPORTED


def test_isosurface_normals_refusals():
    lo = (C.c_float * 3)(0, 0, 0)
    hi = (C.c_float * 3)(1, 1, 1)
    nrm = _cabi.lib().mipnerf_b200_isosurface_normals
    assert nrm(FAKE, 4, 1, 2, lo, hi, 0.0, FAKE, FAKE, None) == _cabi.EINVAL
    assert nrm(None, 4, 3, 2, lo, hi, 0.0, FAKE, FAKE, None) == _cabi.EINVAL
    assert nrm(FAKE, 4, 3, 2, None, hi, 0.0, FAKE, FAKE, None) == _cabi.EINVAL
    assert nrm(FAKE, 4, 3, 2, lo, None, 0.0, FAKE, FAKE, None) == _cabi.EINVAL
    assert nrm(FAKE, 4, 3, 2, lo, hi, 0.0, None, FAKE, None) == _cabi.EINVAL


def test_query_radiance_python_shape_checks():
    model = mp.MipNerf()
    with pytest.raises(ValueError):
        model.query_radiance(torch.zeros(4, 3), None, torch.zeros(5, 3))
    with pytest.raises(ValueError):
        model.query_radiance(torch.zeros(4, 3), torch.zeros(4, 2), torch.zeros(4, 3))
    with pytest.raises(ValueError):
        model.query_radiance(torch.zeros(4, 3))  # use_viewdirs=True needs directions
