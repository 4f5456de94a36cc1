"""Baked grids without a GPU: the float64 renderer reference against closed forms, the mask / index / occupancy
builder on hand-made density grids (including the exact-skip invariant, exhaustively on small grids), and the
argument checks of the Python surface and of mipnerf_b200_grid_render."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_render_ref as ref
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi, baked

BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))


def const_levels(n0, sigmas, coeff, degree=0):
    """Levels of constant density sigmas[l], every point kept with SH row `coeff` [K, 3]."""
    out = []
    for lvl, s in enumerate(sigmas):
        n = (n0 - 1) // (1 << lvl) + 1
        idx = np.arange(n ** 3, dtype=np.int32).reshape(n, n, n)
        out.append((np.full((n, n, n), s), idx, np.broadcast_to(coeff, (n ** 3,) + coeff.shape).copy()))
    return out


def rays_inside(b, seed=0):
    """Rays whose [near, far] segment lies inside BOX."""
    g = np.random.default_rng(seed)
    o = g.uniform(-0.4, 0.4, (b, 3))
    d = g.normal(size=(b, 3))
    d *= g.uniform(0.3, 2.0, (b, 1)) / np.linalg.norm(d, axis=1, keepdims=True)
    near = g.uniform(0.0, 0.1, b)
    far = near + 0.5 / np.linalg.norm(d, axis=1) * g.uniform(0.2, 1.0, b)
    return o, d, d / np.linalg.norm(d, axis=1, keepdims=True), near, far


@pytest.mark.parametrize("sigma", [0.0, 0.3, 4.0])
def test_reference_constant_box_acc(sigma):
    o, d, v, near, far = rays_inside(64)
    levels = const_levels(9, [sigma], np.zeros((1, 3)))
    rgb, dist, acc = ref.render(levels, BOX, 0, 0.0, o, d, v, np.zeros(64), near, far, 0.01, False)
    d32 = d.astype(np.float32).astype(np.float64)
    length = (far.astype(np.float32).astype(np.float64) - near.astype(np.float32)) * np.linalg.norm(d32, axis=1)
    want = 1 - np.exp(-sigma * length)
    assert np.max(np.abs(acc - want)) < 1e-6
    # uniform density along the segment: the weights' mean t is that of an exponential restricted to [near, far]
    assert np.all(dist >= near.astype(np.float32) - 1e-6) and np.all(dist <= far.astype(np.float32) + 1e-6)


def test_reference_degree0_constant_colour():
    o, d, v, near, far = rays_inside(64, seed=1)
    coeff = np.array([[0.7, -1.3, 2.1]])
    p = 0.001
    levels = const_levels(9, [2.0], coeff)
    for white in (False, True):
        rgb, _, acc = ref.render(levels, BOX, 0, p, o, d, v, np.zeros(64), near, far, 0.01, white)
        raw = mp.field.SH_C0 * coeff[0]
        p32 = float(np.float32(p))  # the kernel's fp32 rgb_padding
        col = (1 + 2 * p32) / (1 + np.exp(-raw)) - p32
        want = acc[:, None] * col + (1 - acc[:, None] if white else 0.0)
        assert np.max(np.abs(rgb - want)) < 1e-12


def test_reference_integer_level_uses_that_level_alone():
    """Single-sample rays (far - near below one step) at t = 2, 3-level grid of densities 1, 2, 4."""
    n0, s0 = 9, 2.0 / 8
    sig = [1.0, 2.0, 4.0]
    levels = const_levels(n0, sig, np.zeros((1, 3)))
    t = 0.5
    o = np.zeros((4, 3))
    d = np.array([[1.0, 0, 0]] * 4)
    near, far = np.full(4, t - 1e-3), np.full(4, t + 1e-3)
    # lambda = log2(sqrt(3) r t / s0): 0 (clamped from below), exactly 1, exactly 2, above 2 (clamped)
    r = np.array([0.0, 2 * s0 / (np.sqrt(3) * t), 4 * s0 / (np.sqrt(3) * t), 100.0])
    _, _, acc = ref.render(levels, BOX, 0, 0.0, o, d, d, r, near, far, 0.01, False)
    K, dt, dn = ref.sample_lattice(d, near, far, 0.01)
    assert np.all(K == 1)
    delta = dt.astype(np.float64) * dn
    want = 1 - np.exp(-np.array([sig[0], sig[1], sig[2], sig[2]]) * delta)
    assert np.max(np.abs(acc - want) / want) < 1e-9
    # and a lambda of 1.25 blends levels 1 and 2 with weights 3/4, 1/4
    r5 = np.array([2 ** 1.25 * s0 / (np.sqrt(3) * t)])
    _, _, acc5 = ref.render(levels, BOX, 0, 0.0, o[:1], d[:1], d[:1], r5, near[:1], far[:1], 0.01, False)
    assert abs(acc5[0] - (1 - np.exp(-(0.75 * 2 + 0.25 * 4) * delta[0]))) < 1e-12


def test_reference_termination_and_miss():
    o = np.array([[-3.0, 0.1, 0.2], [-3.0, 5.0, 0.0]])
    d = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.0]])
    levels = const_levels(9, [1000.0], np.zeros((1, 3)))
    rgb, dist, acc = ref.render(levels, BOX, 0, 0.0, o, d, d, np.zeros(2), np.full(2, 1.0), np.full(2, 5.0), 0.01, True)
    assert 1 - 1e-4 <= acc[0] <= 1 and acc[1] == 0 and np.all(rgb[1] == 1)
    assert abs(dist[0] - 2.0) < 0.02 and dist[1] == 1.0  # clamp to near


# ---- the mask / index / occupancy builder ----------------------------------------------------------------------

def test_structure_dilation_and_index():
    d = torch.zeros(9, 9, 9)
    d[4, 4, 4] = 5.0
    d[4, 4, 5] = 0.25  # below the threshold but inside the dilation: kept with its density
    d[0, 0, 8] = 0.5   # below and outside: dropped
    (bd,), (idx,), occ = mp.grid_structure([d], threshold=1.0, block=4)
    keep = torch.zeros(9, 9, 9, dtype=torch.bool)
    keep[3:6, 3:6, 3:6] = True
    assert torch.equal(idx >= 0, keep)
    assert torch.equal(idx[keep], torch.arange(27, dtype=torch.int32))  # x-fastest order
    assert torch.equal(bd, torch.where(keep, d, torch.zeros(())))
    assert bd[0, 0, 8] == 0 and bd[4, 4, 5] == 0.25
    assert occ.shape == (2, 2, 2) and occ.dtype == torch.uint8


def test_structure_union_across_levels():
    d0 = torch.zeros(17, 17, 17)
    d1 = torch.zeros(9, 9, 9)
    d1[7, 7, 7] = 3.0  # only level 1 is non-zero: macro cell (1, 1, 1) of block 8 must be occupied
    _, _, occ = mp.grid_structure([d0, d1], threshold=1.0, block=8)
    assert occ[1, 1, 1] == 1 and occ[0, 0, 0] == 0
    _, _, occ_only0 = mp.grid_structure([d0, torch.zeros(9, 9, 9)], threshold=1.0, block=8)
    assert not occ_only0.any()


def _random_sparse(n0, levels, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for lvl in range(levels):
        n = tuple((m - 1) // (1 << lvl) + 1 for m in n0)
        d = torch.rand(n, generator=g) * 5
        d = torch.where(torch.rand(n, generator=g) < 0.02, d, torch.zeros(()))
        d[..., int(0.4 * n[2]):] = 0  # the far side of x empty at every level: empty and occupied cells
        out.append(d)
    return out


@pytest.mark.parametrize("n0,levels,block", [((17, 17, 17), 1, 8), ((25, 17, 33), 2, 8), ((33, 25, 17), 3, 4),
                                              ((33, 33, 41), 3, 8), ((9, 25, 33), 4, 8)])
def test_structure_exact_skip_invariant(n0, levels, block):
    """Every position in an empty macro cell, and positions a few ulp outside it, interpolate to exactly 0 at every
    level: checked at quarter steps of the finest lattice on every axis (cell corners and faces included)."""
    dens = _random_sparse(n0, levels, seed=sum(n0) + levels)
    baked_d, _, occ = mp.grid_structure(dens, threshold=1.0, block=block)
    assert 0 < int(occ.sum()) < occ.numel(), "test grid should have both empty and occupied cells"
    nz, ny, nx = n0
    lo, hi = np.array([-1.5, -1.0, -0.5]), np.array([1.5, 0.5, 2.0])
    step = (hi - lo) / (np.array([nx, ny, nz]) - 1)
    sub = np.linspace(0, block, 4 * block + 1)
    for cz, cy, cx in zip(*np.nonzero(occ.numpy() == 0)):
        cell = np.array([cx, cy, cz])
        axes = []
        for a in range(3):
            u = cell[a] * block + sub
            u = u[u <= [nx, ny, nz][a] - 1]
            u = np.concatenate([u, [u[0] - 1e-6, u[-1] + 1e-6]])  # just outside the cell
            axes.append(lo[a] + np.clip(u, 0, [nx, ny, nz][a] - 1) * step[a])
        x = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
        for lvl, bd in enumerate(baked_d):
            v = ref.trilinear(bd.numpy().astype(np.float64), lo, hi, x)
            assert np.all(v == 0), (lvl, (cx, cy, cz))


def test_structure_refusals():
    with pytest.raises(ValueError):
        mp.grid_structure([torch.zeros(9, 9, 9), torch.zeros(4, 4, 4)], 1.0)  # not nested
    with pytest.raises(ValueError):
        mp.grid_structure([torch.zeros(9, 9, 9)] * 5, 1.0)                     # L > 4
    with pytest.raises(ValueError):
        mp.grid_structure([torch.zeros(17, 17, 17), torch.zeros(9, 9, 9)], 1.0, block=3)


def test_python_argument_checks():
    assert baked.level_resolutions(257, 3) == [(257,) * 3, (129,) * 3, (65,) * 3]
    assert baked.level_resolutions((33, 17, 9), 4) == [(33, 17, 9), (17, 9, 5), (9, 5, 3), (5, 3, 2)]
    for res, lv in ((256, 2), (257, 5), (257, 0), ((33, 18, 9), 2), (35, 3)):
        with pytest.raises(ValueError):
            baked.level_resolutions(res, lv)
    with pytest.raises(ValueError):
        mp.bake_grid(None, 33, levels=1, degree=4)
    with pytest.raises(ValueError):
        mp.bake_grid(None, 33, levels=5)
    with pytest.raises(ValueError):
        mp.bake_grid(None, 34, levels=2)
    d, i, o = torch.zeros(9, 9, 9), torch.full((9, 9, 9), -1, dtype=torch.int32), torch.zeros(1, 1, 1)
    with pytest.raises(ValueError):
        mp.BakedGrid([d], [i], [torch.zeros(0, 25, 3)], o, degree=4)
    with pytest.raises(ValueError):
        mp.BakedGrid([d], [i], [torch.zeros(0, 9, 3)], o, degree=1)  # coefficient count of degree 2


# ---- refusals of the C ABI (every one is decided before anything launches) --------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def _valid_args():
    """A well-formed grid / rays description on dummy (never dereferenced) addresses."""
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(0x1000, 0x2000, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(0x3000, 0x4000, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    return g, r


@pytest.mark.parametrize("case", ["grid_null", "rays_null", "origins_null", "viewdirs_null", "rgb_null", "acc_null",
                                  "cells_null", "occupancy_null", "step_zero", "step_negative", "step_nan",
                                  "degree_4", "degree_neg", "levels_0", "levels_5", "block_odd", "not_nested",
                                  "bounds_empty", "negative_rays"])
def test_cabi_refusals(lib, case):
    g, r = _valid_args()
    step, out = 0.01, [0xC000, 0xD000, 0xE000]
    gp, rp = C.byref(g), C.byref(r)
    if case == "grid_null":
        gp = None
    elif case == "rays_null":
        rp = None
    elif case == "origins_null":
        r.origins = None
    elif case == "viewdirs_null":
        r.viewdirs = None
    elif case == "rgb_null":
        out[0] = None
    elif case == "acc_null":
        out[2] = None
    elif case == "cells_null":
        g.levels[1].cells = None
    elif case == "occupancy_null":
        g.occupancy = None
    elif case.startswith("step"):
        step = {"step_zero": 0.0, "step_negative": -0.1, "step_nan": float("nan")}[case]
    elif case == "degree_4":
        g.degree = 4
    elif case == "degree_neg":
        g.degree = -1
    elif case == "levels_0":
        g.num_levels = 0
    elif case == "levels_5":
        g.num_levels = 5
    elif case == "block_odd":
        g.block = 3
    elif case == "not_nested":
        g.levels[1].ny = 8
    elif case == "bounds_empty":
        g.hi[1] = -1.0
    elif case == "negative_rays":
        r.num_rays = -1
    rc = lib.mipnerf_b200_grid_render(gp, rp, step, 1, *out, None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


MARCHING = ["grid_render", "grid_render_u8", "grid_render_bricks", "grid_render_backward", "grid_visibility",
            "grid_visibility_bricks"]
_RENDERS, _BRICKS = MARCHING[:3], ("grid_render_bricks", "grid_visibility_bricks")


def _march_refusal(lib, name, faults):
    """The message `name` refuses a valid argument set with `faults` applied; a fault an entry point has no argument
    for is not applied."""
    g, r = _valid_args()
    step, out = 0.01, [0xC000, 0xD000, 0xE000]
    bricks, sh = _cabi.GridBricks(), _cabi.GridShU8()
    for lvl in range(2):
        if name in _BRICKS:
            g.levels[lvl].cells = None
            bricks.table[lvl], bricks.pool[lvl] = 0x10000 + lvl, 0x20000 + lvl
        if name in ("grid_render_u8", "grid_render_bricks"):
            g.levels[lvl].sh = None
            sh.rows[lvl] = 0x30000 + lvl
    grads, mw = _cabi.GridGrads(), (C.c_void_p * 2)(0xF000, 0xF100)
    grads.density[:2], grads.sh[:2] = [0x40000, 0x40100], [0x50000, 0x50100]
    gp, rp, bp, sp, gr = C.byref(g), C.byref(r), C.byref(bricks), C.byref(sh), C.byref(grads)
    for f in faults:
        if f == "grid":
            gp = None
        elif f == "origins":
            r.origins = None
        elif f == "viewdirs":
            r.viewdirs = None
        elif f == "num_rays":
            r.num_rays = -1
        elif f == "rgb":
            out[0] = None
        elif f == "step":
            step = 0.0
        elif f == "bricks":
            bp = None
        elif f == "degree":
            g.degree = 4
        elif f == "sh":
            sp = None
        elif f == "grads":
            gr = None
        elif f == "max_weight":
            mw = None
    call = {"grid_render": lambda: lib.mipnerf_b200_grid_render(gp, rp, step, 1, *out, None),
            "grid_render_u8": lambda: lib.mipnerf_b200_grid_render_u8(gp, sp, rp, step, 1, *out, None),
            "grid_render_bricks": lambda: lib.mipnerf_b200_grid_render_bricks(gp, bp, None, rp, step, 1, *out, None),
            "grid_render_backward": lambda: lib.mipnerf_b200_grid_render_backward(gp, rp, step, 1, 0x60000, None,
                                                                                  None, gr, None),
            "grid_visibility": lambda: lib.mipnerf_b200_grid_visibility(gp, rp, step, mw, None),
            "grid_visibility_bricks": lambda: lib.mipnerf_b200_grid_visibility_bricks(gp, bp, rp, step, mw, None)}[name]
    assert call() == _cabi.EINVAL, (name, faults)
    return _cabi.last_error()


STEP_MSG = "step=0: need a finite step > 0"
DEGREE_MSG = "degree=4: need 0..3"


@pytest.mark.parametrize("faults,want", [
    (("grid", "origins"), {n: "grid is NULL" for n in MARCHING}),
    (("num_rays", "grid"), {n: "grid is NULL" for n in MARCHING}),
    (("origins", "viewdirs"), {n: "a ray field is NULL" for n in MARCHING}),
    (("num_rays", "viewdirs"), {n: "num_rays=-1" for n in MARCHING}),
    (("viewdirs", "rgb"), {n: "rays->viewdirs is NULL" for n in MARCHING}),
    (("bricks", "viewdirs"), {n: "rays->viewdirs is NULL" for n in MARCHING}),
    (("rgb", "step"), {n: "rgb / distance / acc is NULL" if n in _RENDERS else STEP_MSG for n in MARCHING}),
    (("step", "bricks"), {n: STEP_MSG for n in MARCHING}),
    (("bricks", "degree"), {n: "bricks is NULL" if n in _BRICKS else DEGREE_MSG for n in MARCHING}),
    (("degree", "sh"), {n: DEGREE_MSG for n in MARCHING}),
    (("degree", "grads"), {n: DEGREE_MSG for n in MARCHING}),
    (("degree", "max_weight"), {n: DEGREE_MSG for n in MARCHING}),
    (("sh", "max_weight"), {**{n: None for n in MARCHING}, "grid_render_u8": "sh is NULL",
                            "grid_visibility": "max_weight is NULL", "grid_visibility_bricks": "max_weight is NULL"}),
])
def test_marching_refusal_order(lib, faults, want):
    """Every entry point that marches rays refuses the first of two faults in one order: grid, rays, viewdirs, the
    outputs, the step, bricks, the grid description, then what the entry point checks on its own."""
    for name in MARCHING:
        if want[name] is not None:
            assert _march_refusal(lib, name, faults) == want[name], (name, faults)


def test_kernel_registered_with_profiler(lib):
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-1] == "grid_render"
