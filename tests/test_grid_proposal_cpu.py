"""Proposal sampling from a baked grid without a GPU: the float64 reference (tests/grid_proposal_ref.py) against the
closed form of a constant-density slab, the argument checks of mipnerf_b200_grid_proposal and
mipnerf_b200_forward_proposed(_rng) in the order they refuse, the new profiler id's position, and the Python
refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_proposal_ref as pref
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi
from mipnerf_pl_b200.rays import Rays


# ---- the reference ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sigma", [0.0, 0.5, 2.0, 40.0])
@pytest.mark.parametrize("levels", [1, 2])
def test_reference_constant_slab(sigma, levels):
    """Density sigma on the whole lattice of [-1, 1]^3 and 0 outside it: along +x from inside, intervals of exact fp32
    length 1/8 give w_i = e^{-sigma delta i} (1 - e^{-sigma delta}) up to the box face, then 0.  With two levels the
    blend of two constant lattices is the same constant."""
    dens = [np.full((n, n, n), sigma) for n in (17, 9)[:levels]]
    bounds = ((-1.0,) * 3, (1.0,) * 3)
    o = np.array([[-0.875, 0.1, -0.2], [-0.875, 0.1, -0.2]], np.float32)
    d = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.0]], np.float32)
    radii = np.array([0.0, 0.05], np.float32)  # lambda 0, and a level blend
    t = np.tile(np.arange(25, dtype=np.float32) / 8, (2, 1))  # x = -0.875 .. 2.125
    w, sens = pref.proposal(dens, bounds, o, d, radii, t)
    delta = 1 / 8
    inside = -0.875 + (np.arange(24) + 0.5) / 8 <= 1.0
    want = np.where(inside, np.exp(-sigma * delta * np.arange(24)) * (1 - np.exp(-sigma * delta)), 0.0)
    np.testing.assert_allclose(w, np.tile(want, (2, 1)), rtol=1e-12, atol=1e-300)
    assert np.all(sens == 0.0)


def test_reference_weights_are_volumetric_rendering():
    """A random lattice: the weights composite to 1 - exp(-total depth), and a degenerate interval (t_i = t_{i+1})
    and a ray with near == far get weight 0."""
    g = np.random.default_rng(0)
    dens = [4.0 * g.random((9, 9, 9)), 4.0 * g.random((5, 5, 5))]
    o = np.array([[-2.0, 0.1, 0.3], [0.2, 0.2, 0.2]], np.float32)
    d = np.array([[1.0, 0.05, -0.1], [0.0, 1.0, 0.0]], np.float32)
    t = np.sort(g.uniform(0.5, 3.5, (2, 33)).astype(np.float32), axis=1)
    t[0, 5] = t[0, 4]
    t[1] = 1.25
    w, _ = pref.proposal(dens, ((-1.0,) * 3, (1.0,) * 3), o, d, np.array([0.01, 0.02], np.float32), t)
    assert w[0, 4] == 0.0 and np.all(w[1] == 0.0)
    assert np.all(w >= 0) and w[0].sum() < 1


# ---- the C ABI --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def _grid_args(bricked=False):
    """A well-formed two-level grid, rays and optional bricks on dummy (never dereferenced) addresses."""
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(None if bricked else 0x1000, 0x2000, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(None if bricked else 0x3000, 0x4000, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    b = _cabi.GridBricks()
    b.table[0], b.table[1] = 0x10000, 0x10100
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    return g, b, r


def _proposal_refusal(lib, faults, bricked=False):
    g, b, r = _grid_args(bricked)
    gp, bp, rp = C.byref(g), C.byref(b) if bricked else None, C.byref(r)
    t, w, n = 0xC000, 0xD000, 128
    for f in faults:
        if f == "grid":
            gp = None
        elif f == "rays":
            rp = None
        elif f == "origins":
            r.origins = None
        elif f == "num_rays":
            r.num_rays = -1
        elif f == "t_samples":
            t = None
        elif f == "weights":
            w = None
        elif f == "n0":
            n = 0
        elif f == "n257":
            n = 257
        elif f == "cells":
            g.levels[1].cells = 0x3000
        elif f == "table":
            b.table[1] = None
        elif f == "degree":
            g.degree = 4
        elif f == "occupancy":
            g.occupancy = None
        elif f == "not_nested":
            g.levels[1].nx = 8
    assert lib.mipnerf_b200_grid_proposal(gp, bp, rp, t, n, w, None) == _cabi.EINVAL, faults
    return _cabi.last_error()


@pytest.mark.parametrize("faults,want", [
    (("grid", "origins"), "grid is NULL"),
    (("rays", "t_samples"), "rays is NULL"),
    (("origins", "t_samples"), "a ray field is NULL"),
    (("num_rays", "weights"), "num_rays=-1"),
    (("t_samples", "n0"), "t_samples / weights is NULL"),
    (("weights", "degree"), "t_samples / weights is NULL"),
    (("n0", "degree"), "num_samples=0: need 1..256"),
    (("n257", "occupancy"), "num_samples=257: need 1..256"),
    (("degree",), "degree=4: need 0..3"),
    (("occupancy",), "occupancy is NULL"),
    (("not_nested",), "level 1: 8 x 9 x 9 points, need >= 2 per axis and (n_0 - 1) / 2^1 + 1"),
])
def test_proposal_refusal_order(lib, faults, want):
    """Refusals in order: grid, rays, t_samples / weights, num_samples, then the grid description."""
    assert _proposal_refusal(lib, faults) == want


def test_proposal_brick_refusals(lib):
    """With bricks, the cells are the bricks, as for the _bricks entry points; without, the dense cells are needed."""
    assert _proposal_refusal(lib, ("cells",), bricked=True) == \
        "level 1: levels[1].cells is set; the cells are read from bricks"
    assert _proposal_refusal(lib, ("table",), bricked=True) == "level 1: bricks->table[1] is NULL"
    assert _proposal_refusal(lib, ("t_samples", "table"), bricked=True) == "t_samples / weights is NULL"
    g, _, r = _grid_args(bricked=True)
    assert lib.mipnerf_b200_grid_proposal(C.byref(g), None, C.byref(r), 0xC000, 128, 0xD000, None) == _cabi.EINVAL
    assert _cabi.last_error() == "level 0: cells is NULL"


def test_proposal_without_rays_launches_nothing(lib):
    """No ray: NULL fenceposts and weights are accepted and nothing is launched, so the call succeeds without a device."""
    g, _, r = _grid_args()
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_proposal(C.byref(g), None, C.byref(r), None, 128, None, None) == _cabi.OK


def _forward_args(levels=2):
    cfg = mp.MipNerf(num_levels=levels)._config()
    lin = (_cabi.Linear * 12)()
    shapes = [(96, 256), (256, 256), (256, 256), (256, 256), (256, 256), (352, 256), (256, 256), (256, 256),
              (256, 1), (256, 256), (283, 128), (128, 3)]
    for i, (k, m) in enumerate(shapes):
        lin[i] = _cabi.Linear(0x100000 + 0x1000 * i, 0x200000 + 0x1000 * i, k, m)
    w = _cabi.Weights(lin, 12, -1, None, 0)
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    outs = (_cabi.LevelOut * 3)()
    for i in range(3):
        outs[i] = _cabi.LevelOut(0x300000 + i, 0x310000 + i, 0x320000 + i, None, None, None, None)
    return cfg, w, r, outs


def _forward_refusal(lib, faults, rng_form):
    cfg, w, r, outs = _forward_args()
    cp, wp, rp, op = C.byref(cfg), C.byref(w), C.byref(r), outs
    t_prev, w_prev, randomized, u_jitter, ws, nbytes = 0xC000, 0xD000, 0, None, 0xE000, 1 << 40
    rng = _cabi.Rng(1, 0)
    rngp = C.byref(rng)
    for f in faults:
        if f == "config":
            cp = None
        elif f == "levels":
            cfg.num_levels = 1
        elif f == "samples":
            cfg.num_samples = 100
        elif f == "weights":
            w.num_linears = 11
        elif f == "rays":
            r.origins = None
        elif f == "outs":
            op = None
        elif f == "t_prev":
            t_prev = None
        elif f == "w_prev":
            w_prev = None
        elif f == "viewdirs":
            r.viewdirs = None
        elif f == "u_jitter":
            randomized = 1
        elif f == "comp_rgb":
            outs[0].comp_rgb = None
        elif f == "workspace":
            ws = None
        elif f == "rng":
            rngp = None
    if rng_form:
        rc = lib.mipnerf_b200_forward_proposed_rng(cp, wp, rp, t_prev, w_prev, rngp, 1, _cabi.FP32, op, ws, nbytes,
                                                   None)
    else:
        rc = lib.mipnerf_b200_forward_proposed(cp, wp, rp, t_prev, w_prev, randomized, u_jitter, 1, _cabi.FP32, op,
                                               ws, nbytes, None)
    assert rc != _cabi.OK, faults
    return rc, _cabi.last_error()


@pytest.mark.parametrize("rng_form", [False, True])
@pytest.mark.parametrize("faults,code,want", [
    (("config", "levels"), _cabi.EINVAL, "config is NULL"),
    (("samples", "levels"), _cabi.EUNSUPPORTED, "num_samples=100: need a multiple of 32 in {32,64,96,128,192,256}"),
    (("levels", "weights"), _cabi.EINVAL, "num_levels=1: a forward from proposal weights needs >= 2 levels"),
    (("weights", "rays"), _cabi.EINVAL, "expected 12 linears (state_dict order), got 11"),
    (("rays", "outs"), _cabi.EINVAL, "a ray field is NULL"),
    (("outs", "t_prev"), _cabi.EINVAL, "outs is NULL"),
    (("t_prev", "viewdirs"), _cabi.EINVAL, "t_prev / w_prev is NULL"),
    (("w_prev", "viewdirs"), _cabi.EINVAL, "t_prev / w_prev is NULL"),
    (("viewdirs", "comp_rgb"), _cabi.EINVAL, "use_viewdirs but rays.viewdirs is NULL"),
    (("comp_rgb", "workspace"), _cabi.EINVAL, "outs[0] misses comp_rgb/distance/acc"),
])
def test_forward_proposed_refusal_order(lib, faults, code, want, rng_form):
    """Both forms refuse in one order: the config, num_levels, the weights, the rays, outs, t_prev / w_prev, then the
    forward's own checks."""
    assert _forward_refusal(lib, faults, rng_form) == (code, want)


def test_forward_proposed_draw_refusals(lib):
    """randomized=1 needs u_jitter (no t_rand: level 0 is not run); the _rng form needs its generator; the workspace
    rule is the forward's."""
    rc, msg = _forward_refusal(lib, ("u_jitter",), False)
    assert rc == _cabi.EINVAL and msg.startswith("randomized=1 needs u_jitter")
    assert _forward_refusal(lib, ("rng", "config"), True) == (_cabi.EINVAL, "rng is NULL")
    rc, msg = _forward_refusal(lib, ("workspace",), False)
    assert rc == _cabi.EWORKSPACE and msg.startswith("workspace 1099511627776 < ")


def test_symbols_and_profiler_id(lib):
    for name in ("mipnerf_b200_grid_proposal", "mipnerf_b200_forward_proposed", "mipnerf_b200_forward_proposed_rng"):
        assert name in _cabi.EXPORTED_SYMBOLS and hasattr(lib, name)
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-8:] == ["grid_proposal", "grid_tv", "grid_visibility_bricks", "grid_render_bricks",
                          "grid_render_backward", "grid_render_u8", "grid_visibility", "grid_render"]
    assert names.count("grid_proposal") == 1
    assert lib.mipnerf_b200_abi_version() == 4


# ---- Python refusals --------------------------------------------------------------------------------------------

def _cpu_grid():
    d = torch.zeros(9, 9, 9)
    d[4, 4, 4] = 1.0
    baked, idx, occ = mp.grid_structure([d], threshold=0.5)
    return mp.BakedGrid(baked, idx, [torch.zeros(int((idx[0] >= 0).sum()), 1, 3)], occ, degree=0)


def _cpu_rays(n=4):
    z = torch.zeros(n, 3)
    one = torch.ones(n, 1)
    return Rays(z, z + 1, z + 1, one, one, one, 2 * one)


def test_python_refusals():
    grid = _cpu_grid()
    with pytest.raises(ValueError, match="num_levels=1"):
        mp.MipNerf(num_levels=1).forward_proposed(_cpu_rays(), grid, False, True)
    with pytest.raises(NotImplementedError):
        mp.MipNerf(ray_shape="cylinder").forward_proposed(_cpu_rays(), grid, False, True)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        mp.MipNerf().forward_proposed(_cpu_rays(), grid, False, True)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        grid.proposal(_cpu_rays(), torch.zeros(4, 129))
