"""The streamed sparse bake without a GPU: `sparse_grid_structure` on analytic density callbacks against
`grid_structure` -> dense BakedGrid -> `sparsify()` in every array (1-4 levels, axes that are not multiples of 8 and
non-cubic, slabs from one brick layer to the whole level), the int32 row-count refusal, the quantize codec shared by
`BakedGrid.quantize` and the streamed bake, and `tools/bake_grid.py`'s choice of path."""
import numpy as np
import pytest
import torch

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import baked
from tools import bake_grid as bake_tool

BOX = ((-1.0, -0.75, -1.25), (1.0, 1.25, 0.75))


def lattice_density(kind, res, seed=0):
    """[nz, ny, nx] fp32 densities of an analytic scene on a lattice (nx, ny, nz) over [-1, 1]^3."""
    nx, ny, nz = res
    z, y, x = torch.meshgrid(*[torch.linspace(-1.0, 1.0, n) for n in (nz, ny, nx)], indexing="ij")
    if kind == "shells":
        r = torch.sqrt(x * x + y * y + z * z)
        near = ((r - 0.45).abs() < 0.06) | ((r - 0.8).abs() < 0.04)
        return torch.where(near, 2.0 + r, torch.zeros(()))
    if kind == "point":  # one point above the threshold, off-centre
        d = torch.zeros(nz, ny, nx)
        d[nz // 3, ny - 2, 1] = 5.0
        return d
    if kind == "empty":
        return torch.zeros(nz, ny, nx)
    if kind == "full":
        return 0.5 + torch.rand(nz, ny, nx, generator=torch.Generator().manual_seed(seed))
    if kind == "at_threshold":  # exactly the threshold (not kept) beside points just above it
        d = torch.full((nz, ny, nx), 1.0)
        d[::5, ::3, ::4] = float(np.nextafter(np.float32(1.0), np.float32(2.0)))
        d[:, :, nx // 2:] = 1.0
        return d
    raise ValueError(kind)


THRESHOLD = {"shells": 1.0, "point": 1.0, "empty": 1.0, "full": 0.0, "at_threshold": 1.0}


def dense_then_sparse(dens, threshold, block, degree=1, seed=0):
    bd, idx, occ = mp.grid_structure(dens, threshold, block)
    g = torch.Generator().manual_seed(seed)
    sh = [torch.randn(int((i >= 0).sum()), (degree + 1) ** 2, 3, generator=g) for i in idx]
    return mp.BakedGrid(bd, idx, sh, occ, BOX, degree, 0.001, block).sparsify(), idx


def assert_stream_equals_dense(kind, res0, levels, slab, block=None):
    res = mp.baked.level_resolutions(res0, levels)
    dens = [lattice_density(kind, r, seed=lvl) for lvl, r in enumerate(res)]
    block = block or max(8, 1 << (levels - 1))
    calls = []

    def density_fn(lvl, z0, z1):
        calls.append((lvl, z0, z1))
        return dens[lvl][z0:z1].clone()

    tables, pools, positions, occ = mp.sparse_grid_structure(density_fn, res0, levels, THRESHOLD[kind], block, slab)
    want, idx = dense_then_sparse(dens, THRESHOLD[kind], block)
    assert occ.dtype == torch.uint8 and torch.equal(occ, want.occupancy)
    for lvl, ((t, p), (u, q)) in enumerate(zip(zip(tables, pools), want.bricks)):
        assert t.dtype == u.dtype and torch.equal(t, u), (kind, res0, levels, slab, lvl)
        assert p.dtype == q.dtype and torch.equal(p, q), (kind, res0, levels, slab, lvl)
        flat = (idx[lvl].reshape(-1) >= 0).nonzero().reshape(-1)
        assert positions[lvl].dtype == torch.int64 and torch.equal(positions[lvl], flat)
    # every query is one slab plus at most one layer of halo per side, clipped at the lattice ends
    for lvl, z0, z1 in calls:
        nz = res[lvl][2]
        assert 0 <= z0 < z1 <= nz and z1 - z0 <= 8 * (slab or -(-nz // 8)) + 2
    return tables


LEVEL_CASES = [(25, 1), (33, 2), (49, 3), (65, 4), ((17, 41, 9), 1), ((41, 9, 33), 3), ((129, 17, 25), 2)]


@pytest.mark.parametrize("kind", sorted(THRESHOLD))
@pytest.mark.parametrize("res0,levels", LEVEL_CASES)
def test_stream_equals_dense_sparsify(kind, res0, levels):
    nz = mp.baked.level_resolutions(res0, levels)[0][2]
    for slab in sorted({1, 2, 3, -(-nz // 8)}) + [None]:
        assert_stream_equals_dense(kind, res0, levels, slab)


@pytest.mark.parametrize("nz", [15, 16, 17, 23, 24, 25])
def test_slab_edges_on_every_halo_case(nz):
    """Slab faces at a lattice end, one layer before it, on it and one past a brick face: the last slab holds 7, 8, 1
    or 0 layers past a multiple of 8, so the halo is clipped on either side or on both."""
    for kind in ("shells", "full", "at_threshold"):
        for slab in (1, 2, None):
            assert_stream_equals_dense(kind, (9, 13, nz), 1, slab)


def test_lone_point_in_every_slab_position():
    """One point above the threshold on every z layer in turn: its dilation crosses the slab faces at z = 8k - 1 and
    8k from either side."""
    res = (11, 10, 26)
    for zp in range(26):
        d = torch.zeros(26, 10, 11)
        d[zp, 4, 5] = 3.0
        tables, pools, _, occ = mp.sparse_grid_structure(lambda lvl, z0, z1: d[z0:z1], res, 1, 1.0, 8, 1)
        want, _ = dense_then_sparse([d], 1.0, 8)
        assert torch.equal(tables[0], want.bricks[0][0]) and torch.equal(pools[0], want.bricks[0][1]), zp
        assert torch.equal(occ, want.occupancy), zp


def test_refuses_beyond_int32_rows(monkeypatch):
    res = (9, 9, 25)
    d = torch.full((25, 9, 9), 2.0)
    monkeypatch.setattr(baked, "_MAX_ROWS", 9 * 9 * 25)
    mp.sparse_grid_structure(lambda lvl, z0, z1: d[z0:z1], res, 1, 1.0, 8, 1)  # exactly the limit: fine
    monkeypatch.setattr(baked, "_MAX_ROWS", 9 * 9 * 25 - 1)
    with pytest.raises(ValueError, match="int32"):
        mp.sparse_grid_structure(lambda lvl, z0, z1: d[z0:z1], res, 1, 1.0, 8, 1)


def test_argument_checks():
    d = lambda lvl, z0, z1: torch.zeros(z1 - z0, 9, 9)  # noqa: E731
    with pytest.raises(ValueError, match="block"):
        mp.sparse_grid_structure(d, 9, 2, 1.0, 3)
    with pytest.raises(ValueError, match="slab"):
        mp.sparse_grid_structure(d, 9, 1, 1.0, 8, 0)
    with pytest.raises(ValueError, match="divisible"):
        mp.sparse_grid_structure(d, 10, 2, 1.0, 8)
    with pytest.raises(ValueError, match="shape"):
        mp.sparse_grid_structure(lambda lvl, z0, z1: torch.zeros(z1 - z0, 9, 8), 9, 1, 1.0, 8)


def reference_codec(c):
    """The codec as `BakedGrid.quantize` wrote it before it moved into one function."""
    nc = c.shape[1]
    if c.shape[0] == 0:
        return torch.empty(0, nc, 3, dtype=torch.uint8), torch.zeros(nc, 3), torch.zeros(nc, 3)
    offset, hi = c.amin(dim=0), c.amax(dim=0)
    scale = (hi - offset) / torch.full_like(hi, 255.0)
    live = scale > 0
    code = torch.round((c - offset) / torch.where(live, scale, torch.ones(())))
    return torch.where(live, code.clamp(0, 255), torch.zeros(())).to(torch.uint8), scale, offset


@pytest.mark.parametrize("chunk", [1, 7, 1 << 20])
@pytest.mark.parametrize("degree", [0, 2, 3])
def test_quantize_codec_unchanged(degree, chunk):
    g = torch.Generator().manual_seed(degree)
    nc = (degree + 1) ** 2
    for m in (0, 1, 5, 300):
        c = 3.0 * torch.randn(m, nc, 3, generator=g)
        if m:
            c[:, 0, 1] = 0.25  # a constant column
        q, s, o = baked._quantize_rows(c, 0, chunk)
        rq, rs, ro = reference_codec(c)
        assert q.dtype == torch.uint8 and torch.equal(q, rq) and torch.equal(s, rs) and torch.equal(o, ro)
    bad = torch.zeros(2, nc, 3)
    bad[1, 0, 0] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        baked._quantize_rows(bad, 1)


def test_quantize_uses_the_codec():
    bd, idx, occ = mp.grid_structure([lattice_density("shells", (17, 17, 17))], 1.0, 8)
    sh = [torch.randn(int((idx[0] >= 0).sum()), 4, 3, generator=torch.Generator().manual_seed(1))]
    q = mp.BakedGrid(bd, idx, sh, occ, BOX, 1, 0.001, 8).quantize()
    rq, rs, ro = reference_codec(sh[0])
    assert torch.equal(q.sh[0], rq) and torch.equal(q.sh_scale[0], rs) and torch.equal(q.sh_offset[0], ro)


def test_bake_tool_path_choice():
    args = lambda *a: bake_tool.parse_args(["--ckpt", "c", "--out", "o", *a])  # noqa: E731
    assert bake_tool.streamed(args("--sparse"))
    assert bake_tool.streamed(args("--sparse", "--quantize"))
    assert not bake_tool.streamed(args())
    assert not bake_tool.streamed(args("--quantize"))
    assert not bake_tool.streamed(args("--sparse", "--prune", "data"))
    a = args("--sparse", "--resolution", "65", "33", "17", "--stream-points", "4096")
    assert a.resolution == [65, 33, 17] and a.stream_points == 4096
