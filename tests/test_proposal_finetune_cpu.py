"""Training a baked grid as a proposal, without a GPU: the float64 references of the interlevel loss
(tests/interlevel_ref.py) and of the proposal weights' density gradient (tests/grid_proposal_grad_ref.py) against
closed forms and float64 finite differences, the argument checks of the three new entry points in the order they
refuse, the new profiler ids' positions, and the Python refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_proposal_grad_ref as gref
import grid_proposal_ref as pref
import interlevel_ref as iref
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi
from test_grid_proposal_cpu import _cpu_grid, _cpu_rays, _grid_args

EPS = iref.EPS


# ---- the interlevel reference -----------------------------------------------------------------------------------

def test_interlevel_one_proposal_interval_covers_all():
    """M = 1 with t_hat spanning every fine fencepost: bound_i = w_hat_0 for every i."""
    g = np.random.default_rng(0)
    t = np.sort(g.uniform(2, 6, (3, 34)), axis=1).astype(np.float32)
    w = g.uniform(0, 0.2, (3, 33))
    wh = np.array([[0.05], [0.1], [1.0]])
    th = np.array([[1.0, 7.0]] * 3, np.float32)
    loss, grad, lo, hi = iref.interlevel(t, w, th, wh)
    excess = np.maximum(0, w - wh)
    np.testing.assert_allclose(loss, (excess ** 2 / (w + EPS)).sum(1), rtol=1e-14)
    np.testing.assert_allclose(grad[:, 0], (-2 * excess / (w + EPS)).sum(1), rtol=1e-14)
    assert np.all(lo == 0) and np.all(hi == 1) and loss[2] == 0 and grad[2, 0] == 0


def test_interlevel_disjoint_ranges():
    """Fine intervals wholly before or after t_hat have bound 0: loss sum w^2 / (w + eps), and no gradient."""
    w = np.array([[0.3, 0.0, 0.5], [0.3, 0.0, 0.5]])
    t = np.array([[0.0, 0.5, 0.7, 1.0], [5.0, 5.5, 5.7, 6.0]], np.float32)
    th = np.array([[2.0, 3.0, 4.0], [2.0, 3.0, 4.0]], np.float32)
    loss, grad, lo, hi = iref.interlevel(t, w, th, np.full((2, 2), 0.9))
    np.testing.assert_allclose(loss, [(w[0] ** 2 / (w[0] + EPS)).sum()] * 2, rtol=1e-14)
    assert np.all(grad == 0)
    assert np.all(hi <= lo) and np.all(lo[0] == 0) and np.all(lo[1] == 2)


def test_interlevel_ties():
    """Fine fenceposts equal to the proposal's: interval i is bounded by w_hat_i alone.  A fencepost tie counts the
    proposal interval starting there (t_hat_k <= t_i) and not the one ending there (t_hat_k < t_{i+1}).  A zero-length
    fine interval at a tie takes no proposal interval."""
    g = np.random.default_rng(1)
    t = np.sort(g.uniform(2, 6, (4, 9)), axis=1).astype(np.float32)
    w, wh = g.uniform(0, 0.3, (4, 8)), g.uniform(0, 0.3, (4, 8))
    loss, grad, lo, hi = iref.interlevel(t, w, t, wh)
    excess = np.maximum(0, w - wh)
    # C_{i+1} - C_i is w_hat_i up to the rounding of the running sum
    np.testing.assert_allclose(loss, (excess ** 2 / (w + EPS)).sum(1), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(grad, -2 * excess / (w + EPS), rtol=1e-12, atol=1e-13)
    assert np.all(lo == np.arange(8)) and np.all(hi == np.arange(1, 9))
    tz = np.array([[2.0, 3.0, 3.0, 4.0]], np.float32)  # interval 1 has zero length at the tie t = 3
    _, _, lo, hi = iref.interlevel(tz, np.ones((1, 3)), np.array([[2.0, 3.0, 4.0]], np.float32), np.ones((1, 2)))
    assert lo.tolist() == [[0, 1, 1]] and hi.tolist() == [[1, 1, 2]]


def test_interlevel_finite_differences():
    g = np.random.default_rng(2)
    t = np.sort(g.uniform(2, 6, (5, 40)), axis=1).astype(np.float32)
    th = np.sort(g.uniform(1.5, 6.5, (5, 18)), axis=1).astype(np.float32)
    w, wh = g.uniform(0, 0.2, (5, 39)), g.uniform(0, 0.05, (5, 17))
    _, grad, _, _ = iref.interlevel(t, w, th, wh)
    h = 1e-7
    for j in range(17):
        e = np.zeros_like(wh)
        e[:, j] = h
        fd = (iref.interlevel(t, w, th, wh + e)[0] - iref.interlevel(t, w, th, wh - e)[0]) / (2 * h)
        np.testing.assert_allclose(grad[:, j], fd, rtol=1e-6, atol=1e-9)
    assert np.any(grad != 0)


# ---- the proposal gradient reference ----------------------------------------------------------------------------

def _lattice(g, shapes, keep=1.0):
    dens = [4.0 * g.random(s) * (g.random(s) < keep) for s in shapes]
    index = []
    for d in dens:
        idx = np.full(d.shape, -1, np.int64)
        kept = (d > 0).reshape(-1)
        idx.reshape(-1)[kept] = np.arange(int(kept.sum()))
        index.append(idx)
    return dens, index


@pytest.mark.parametrize("levels", [1, 3])
def test_proposal_grad_finite_differences(levels):
    """The analytic gradient against central differences of grid_proposal_ref's weights, every kept point perturbed in
    turn; random rays across the level blend."""
    g = np.random.default_rng(3 + levels)
    dens, index = _lattice(g, [(9, 9, 9), (5, 5, 5), (3, 3, 3)][:levels], keep=0.6)
    bounds = ((-1.0,) * 3, (1.0,) * 3)
    o = np.array([[-2.0, 0.1, 0.3], [0.2, -2.0, -0.1], [0.3, 0.3, 2.0]], np.float32)
    d = np.array([[1.0, 0.05, -0.1], [0.1, 1.0, 0.05], [-0.05, -0.1, -1.0]], np.float32)
    radii = np.array([0.002, 0.02, 0.05], np.float32)
    t = np.sort(g.uniform(0.5, 3.5, (3, 17)), axis=1).astype(np.float32)
    gw = g.normal(size=(3, 16))
    got = gref.proposal_grad(list(zip(dens, index)), bounds, o, d, radii, t, gw)
    h = 1e-6
    for lvl in range(levels):
        flat = dens[lvl].reshape(-1)
        for p in np.flatnonzero(index[lvl].reshape(-1) >= 0):
            vals = []
            for sign in (1, -1):
                moved = [x.copy() for x in dens]
                moved[lvl].reshape(-1)[p] = flat[p] + sign * h
                vals.append((pref.proposal(moved, bounds, o, d, radii, t)[0] * gw).sum())
            fd = (vals[0] - vals[1]) / (2 * h)
            r = index[lvl].reshape(-1)[p]
            assert abs(got[lvl][r] - fd) <= 1e-6 * max(1.0, abs(fd)), (lvl, r, got[lvl][r], fd)
    assert any(np.any(x != 0) for x in got)


@pytest.mark.parametrize("sigma", [0.5, 2.0])
def test_proposal_grad_total_weight_closed_form(sigma):
    """Constant density sigma on a fully kept lattice, a ray along +x inside it, g = 1: L = 1 - e^{-S_N}, so every
    dL/ds_k = e^{-S_N}, and since the trilinear weights sum to 1 the gradient sums to sum_k delta_k e^{-S_N}."""
    dens = [np.full((9, 9, 9), sigma)]
    index = [np.arange(729).reshape(9, 9, 9)]
    t = (np.arange(13, dtype=np.float32) / 8)[None]  # x = -0.875 .. 0.625
    o, d = np.array([[-0.875, 0.1, -0.2]], np.float32), np.array([[1.0, 0.0, 0.0]], np.float32)
    got = gref.proposal_grad(list(zip(dens, index)), ((-1.0,) * 3, (1.0,) * 3), o, d, np.zeros(1, np.float32), t,
                             np.ones((1, 12)))
    want = 12 * 0.125 * np.exp(-sigma * 12 * 0.125)
    np.testing.assert_allclose(got[0].sum(), want, rtol=1e-12)


def test_proposal_grad_skips_empty_cells():
    """With an occupancy grid, midpoints in its empty macro cells get no gradient; all occupied, the gradient equals
    the one without an occupancy grid."""
    g = np.random.default_rng(7)
    dens, index = _lattice(g, [(17, 17, 17)])
    args = (list(zip(dens, index)), ((-1.0,) * 3, (1.0,) * 3), np.array([[-2.0, 0.05, 0.02]], np.float32),
            np.array([[1.0, 0.0, 0.0]], np.float32), np.zeros(1, np.float32),
            np.linspace(0.5, 3.5, 33, dtype=np.float32)[None], np.ones((1, 32)))
    free = gref.proposal_grad(*args)
    assert np.array_equal(gref.proposal_grad(*args, occupancy=np.ones((2, 2, 2), np.uint8), block=8)[0], free[0])
    occ = np.ones((2, 2, 2), np.uint8)
    occ[:, :, 1] = 0  # x >= 0 empty
    half = gref.proposal_grad(*args, occupancy=occ, block=8)[0]
    pos_x = np.argwhere(index[0] >= 0)[np.argsort(index[0][index[0] >= 0])][:, 2]  # x of each row
    assert np.all(half[pos_x >= 9] == 0) and np.any(free[0][pos_x >= 9] != 0)


# ---- the C ABI --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def _interlevel_refusal(lib, faults, backward):
    args = dict(t=0x1000, w=0x2000, n=128, th=0x3000, wh=0x4000, nh=64, b=5, out=0x5000)
    for f in faults:
        if f == "num_rays":
            args["b"] = -1
        elif f in ("t", "w", "th", "wh", "out"):
            args[f] = None
        elif f == "n0":
            args["n"] = 0
        elif f == "nh0":
            args["nh"] = 0
    a = args
    if backward:
        rc = lib.mipnerf_b200_interlevel_loss_backward(a["t"], a["w"], a["n"], a["th"], a["wh"], a["nh"], a["b"],
                                                       None, 1.0, a["out"], None)
    else:
        rc = lib.mipnerf_b200_interlevel_loss(a["t"], a["w"], a["n"], a["th"], a["wh"], a["nh"], a["b"], a["out"],
                                              None)
    assert rc == _cabi.EINVAL, faults
    return _cabi.last_error()


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("faults,want", [
    (("num_rays", "t"), "num_rays=-1: need >= 0"),
    (("t", "n0"), "NULL tensor"),
    (("wh", "nh0"), "NULL tensor"),
    (("out", "n0"), "NULL tensor"),
    (("n0", "nh0"), "n=0, n_hat=0: need >= 1"),
    (("nh0",), "n=128, n_hat=0: need >= 1"),
])
def test_interlevel_refusal_order(lib, faults, want, backward):
    """Both entry points refuse in one order: num_rays, the NULL tensors, then n / n_hat."""
    assert _interlevel_refusal(lib, faults, backward) == want


def test_interlevel_without_rays_launches_nothing(lib):
    assert lib.mipnerf_b200_interlevel_loss(None, None, 4, None, None, 4, 0, None, None) == _cabi.OK
    assert lib.mipnerf_b200_interlevel_loss_backward(None, None, 4, None, None, 4, 0, None, 1.0, None, None) == _cabi.OK


def _backward_refusal(lib, faults):
    g, _, r = _grid_args()
    gp, rp = C.byref(g), C.byref(r)
    t, dw, n = 0xC000, 0xD000, 128
    gg = _cabi.GridGrads()
    gg.density[0], gg.density[1] = 0xE000, 0xE100
    ggp = C.byref(gg)
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
        elif f == "d_weights":
            dw = None
        elif f == "grads":
            ggp = None
        elif f == "n0":
            n = 0
        elif f == "n257":
            n = 257
        elif f == "cells":
            g.levels[1].cells = None
        elif f == "degree":
            g.degree = 4
        elif f == "density1":
            gg.density[1] = None
    assert lib.mipnerf_b200_grid_proposal_backward(gp, rp, t, n, dw, ggp, None) == _cabi.EINVAL, faults
    return _cabi.last_error()


@pytest.mark.parametrize("faults,want", [
    (("grid", "origins"), "grid is NULL"),
    (("rays", "t_samples"), "rays is NULL"),
    (("origins", "t_samples"), "a ray field is NULL"),
    (("num_rays", "grads"), "num_rays=-1"),
    (("t_samples", "n0"), "t_samples / d_weights / grads is NULL"),
    (("d_weights", "degree"), "t_samples / d_weights / grads is NULL"),
    (("grads", "n257"), "t_samples / d_weights / grads is NULL"),
    (("n0", "degree"), "num_samples=0: need 1..256"),
    (("n257", "cells"), "num_samples=257: need 1..256"),
    (("degree", "density1"), "degree=4: need 0..3"),
    (("cells", "density1"), "level 1: cells is NULL"),
    (("density1",), "level 1 has kept points: grads->density[1] is NULL"),
])
def test_proposal_backward_refusal_order(lib, faults, want):
    """Refusals in order: grid, rays, t_samples / d_weights / grads, num_samples, the (dense) grid, then the
    per-level density gradients."""
    assert _backward_refusal(lib, faults) == want


def test_proposal_backward_without_rays_launches_nothing(lib):
    g, _, r = _grid_args()
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_proposal_backward(C.byref(g), C.byref(r), None, 128, None, None, None) == _cabi.OK


def test_symbols_and_profiler_ids(lib):
    for name in ("mipnerf_b200_interlevel_loss", "mipnerf_b200_interlevel_loss_backward",
                 "mipnerf_b200_grid_proposal_backward"):
        assert name in _cabi.EXPORTED_SYMBOLS and hasattr(lib, name)
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-10:] == ["interlevel_loss", "grid_proposal_backward", "grid_proposal", "grid_tv",
                           "grid_visibility_bricks", "grid_render_bricks", "grid_render_backward", "grid_render_u8",
                           "grid_visibility", "grid_render"]
    assert names.count("interlevel_loss") == 1 and names.count("grid_proposal_backward") == 1
    assert lib.mipnerf_b200_abi_version() == 4


# ---- Python refusals --------------------------------------------------------------------------------------------

def test_interlevel_python_refusals():
    t, w = torch.zeros(4, 9), torch.zeros(4, 8)
    th, wh = torch.zeros(4, 5), torch.zeros(4, 4)
    for bad in ((t[:3], w, th, wh), (t, w[:, :7], th, wh), (t, w, th[:, :4], wh), (t, w, th, wh[:3]),
                (t[:, :1], w[:, :0], th, wh), (t, w, th[:, :1], wh[:, :0]), (t[0], w[0], th[0], wh[0])):
        with pytest.raises(ValueError, match="interlevel_loss"):
            mp.interlevel_loss(*bad)
    with pytest.raises(ValueError, match="one device"):
        mp.interlevel_loss(t, w, th, wh.to("meta"))
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        mp.interlevel_loss(t, w, th, wh)


def test_finetune_proposal_refusals():
    grid = _cpu_grid()
    with pytest.raises(ValueError, match="num_levels=1"):
        mp.finetune_proposal(grid, mp.MipNerf(num_levels=1), None, 1)
    with pytest.raises(NotImplementedError):
        mp.finetune_proposal(grid, mp.MipNerf(ray_shape="cylinder"), None, 1)
    assert not grid.trainable  # refused before the grid was touched
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        grid.requires_grad_().proposal(_cpu_rays(), torch.zeros(4, 129))
