"""The streamed sparse bake on the GPU, on trained-like weights in bf16, fp16x3 and fp32: `density_grid(z_range=...)`
against the whole grid's rows, `bake_grid(sparse=True)` against `bake_grid().sparsify()` in every array (65^3 and
129^3, 1 and 3 levels, degrees 0 and 2, thresholds that keep nothing, a high quantile and everything, slabs from one
brick layer to the whole lattice), the `quantize=True` variants, renders, save / load, and the peak memory against
`bake_grid`'s docstring formula and the dense bake."""
import numpy as np
import pytest
import torch

from helpers import make_state_dict

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"
PRECISIONS = ["bf16", "fp16x3", "fp32"]
_MODELS = {}
_DENSE = {}


def model(precision):
    if precision not in _MODELS:
        m = mp.MipNerf(precision=precision)
        m.load_state_dict(make_state_dict(seed=0, kind="trained_like"))
        _MODELS[precision] = m.to(DEV).eval()
    return _MODELS[precision]


def thresholds(precision):
    """Nothing kept, the 0.9 density quantile, everything kept."""
    q = float(torch.quantile(mp.density_grid(model(precision), 33).flatten(), 0.9))
    return {"empty": 1e30, "q90": q, "full": -1.0}


def dense(precision, res, levels, degree, threshold):
    key = (precision, res, levels, degree, threshold)
    if key not in _DENSE:
        _DENSE.clear()
        _DENSE[key] = mp.bake_grid(model(precision), res, levels, threshold, degree)
    return _DENSE[key]


def assert_same_grid(a, b):
    assert a.sparse and b.sparse and a.quantized == b.quantized
    assert (a.levels, a.degree, a.block, a.bounds) == (b.levels, b.degree, b.block, b.bounds)
    assert np.float32(a.rgb_padding) == np.float32(b.rgb_padding)  # .npz keeps it as float32
    assert a.resolutions == b.resolutions and a.kept == b.kept
    for (t, p), (u, q) in zip(a.bricks, b.bricks):
        assert t.dtype == u.dtype and torch.equal(t, u)
        assert p.dtype == q.dtype and torch.equal(p, q)
    for x, y in zip(a.sh + [a.occupancy], b.sh + [b.occupancy]):
        assert x.dtype == y.dtype and torch.equal(x, y)
    if a.quantized:
        for x, y in zip(a.sh_scale + a.sh_offset, b.sh_scale + b.sh_offset):
            assert torch.equal(x, y)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_density_grid_z_range(precision):
    m = model(precision)
    for res in (65, (33, 17, 41)):
        nz = res if isinstance(res, int) else res[2]
        full = mp.density_grid(m, res)
        for z0, z1 in ((0, nz), (0, 1), (nz - 1, nz), (7, 9), (5, nz - 3), (3, 3)):
            for slab_points in (1 << 22, 3000):  # query chunks that start on other layers than the whole grid's
                part = mp.density_grid(m, res, z_range=(z0, z1), slab_points=slab_points)
                assert part.shape == full[z0:z1].shape and torch.equal(part, full[z0:z1]), (res, z0, z1, slab_points)
    with pytest.raises(ValueError, match="z_range"):
        mp.density_grid(m, 9, z_range=(4, 10))


CASES = [(res, levels, degree) for res in (65, 129) for levels, degree in ((1, 2), (3, 0), (3, 2))]


@pytest.mark.parametrize("res,levels,degree", CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_stream_equals_dense_sparsify(precision, res, levels, degree):
    for name, threshold in thresholds(precision).items():
        want = dense(precision, res, levels, degree, threshold).sparsify()
        if name == "empty":
            assert want.kept == [0] * levels
        if name == "full":
            assert want.kept[0] == res ** 3
        t = -(-res // 8)
        for stream_points in (1, 3 * 512 * t * t, 1 << 30):  # 1 brick layer, 3 layers, the whole lattice
            got = mp.bake_grid(model(precision), res, levels, threshold, degree, sparse=True,
                               stream_points=stream_points)
            assert_same_grid(got, want)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_quantized_variants(precision):
    threshold = thresholds(precision)["q90"]
    m = model(precision)
    base = dense(precision, 65, 3, 2, threshold)
    q = mp.bake_grid(m, 65, 3, threshold, 2, quantize=True)
    want = base.quantize()
    assert q.quantized and not q.sparse
    for x, y in zip(q.cells + q.sh + q.sh_scale + q.sh_offset + [q.occupancy],
                    want.cells + want.sh + want.sh_scale + want.sh_offset + [want.occupancy]):
        assert x.dtype == y.dtype and torch.equal(x, y)
    for stream_points in (1, 1 << 30):
        sq = mp.bake_grid(m, 65, 3, threshold, 2, sparse=True, quantize=True, stream_points=stream_points)
        assert_same_grid(sq, want.sparsify())


def test_renders_and_save_load(tmp_path):
    m = model("bf16")
    threshold = thresholds("bf16")["q90"]
    base = dense("bf16", 65, 3, 2, threshold)
    for quantize in (False, True):
        got = mp.bake_grid(m, 65, 3, threshold, 2, sparse=True, quantize=quantize, stream_points=1)
        ref = base.quantize() if quantize else base
        path = str(tmp_path / f"stream_{quantize}.npz")
        got.save(path)
        back = mp.BakedGrid.load(path, DEV)
        assert_same_grid(back, got)
        for c2w in (mp.spheric_pose(0.4), mp.spheric_pose(2.0, radius=2.5)):
            frames = [mp.render_baked_frame(g, c2w, 128, 128) for g in (got, back, ref)]
            assert float(frames[2][2].max()) > 0
            for a, b, c in zip(*frames):
                assert torch.equal(a, b) and torch.equal(a, c)


def peak_after(fn):
    """(result, largest memory allocated by `fn` beyond what was allocated before it)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated(DEV) - base


@pytest.mark.parametrize("quantize", [False, True])
def test_peak_memory(quantize):
    """129^3, 1 and 3 levels, one brick layer per slab: the transient memory stays under the docstring's bound and
    below the dense bake's."""
    m = model("bf16")
    threshold = thresholds("bf16")["q90"]
    res, degree, slab_points = 129, 2, 1 << 16
    for levels in (1, 3):
        # warm the query workspace at the sizes both bakes use, so it is counted in neither
        mp.bake_grid(m, res, levels, threshold, degree, slab_points=slab_points)
        _DENSE.clear()
        dense_grid, dense_peak = peak_after(lambda: mp.bake_grid(m, res, levels, threshold, degree,
                                                                 slab_points=slab_points, quantize=quantize))
        del dense_grid
        grid, peak = peak_after(lambda: mp.bake_grid(m, res, levels, threshold, degree, slab_points=slab_points,
                                                     sparse=True, quantize=quantize, stream_points=1))
        transient = peak - grid.nbytes
        t = -(-res // 8)
        big_p = (8 + 2) * (8 * t) * (8 * t)
        q = min(big_p, max(1 << 22, res * res))
        nc = (degree + 1) ** 2
        mm, bb = grid.kept, [int(p.shape[0]) for _, p in grid.bricks]
        bound = 8 * sum(mm) + max(64 * big_p + 28 * q + max(8 * a + 4096 * b for a, b in zip(mm, bb)),
                                  (72 + 12 * nc) * slab_points + (12 * nc * (max(mm) + (1 << 19)) if quantize else 0))
        print(f"levels {levels} quantize {quantize}: streamed transient {transient / 2 ** 20:.1f} MiB (bound "
              f"{bound / 2 ** 20:.1f}), dense peak {dense_peak / 2 ** 20:.1f} MiB, grid {grid.nbytes / 2 ** 20:.1f} MiB")
        assert transient <= bound
        assert peak < dense_peak
