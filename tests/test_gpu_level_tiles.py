"""Every CTA of a level-kernel launch hands tiles between its roles: feature buffers and raw-heads buffers alternate
with the tile's index in the CTA, and the weight ring carries on from one tile to the next.  At 256 samples a ray is
two tiles, and a query launch is one 128-point tile per CTA round with a part-filled last tile.  A whole launch must
compute exactly what launches of one ray (one or two tiles) or one 128-point query tile compute.  The batch sizes give
the CTAs one, two or three rays."""
import pytest
import torch

from helpers import make_state_dict

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _model(precision, **kw):
    model = mp.MipNerf(precision=precision, **kw)
    model.load_state_dict(make_state_dict(seed=9, kind="trained_like"))
    return model.to(DEV).eval()


@pytest.mark.parametrize("samples", [128, 256])
@pytest.mark.parametrize("precision", ["bf16", "fp16"])
@pytest.mark.parametrize("extra", ["one_ray", "one", "two", "three"])
def test_forward_matches_single_ray_launches(precision, samples, extra):
    # one CTA of one ray; seven CTAs of one ray; CTA 0 with two rays, the rest one; every CTA two and some three
    b = {"one_ray": 1, "one": 7, "two": _sms() + 1, "three": 2 * _sms() + 5}[extra]
    rays = mp.namedtuple_map(lambda t: t.to(DEV), mp.random_ray_batch(b, seed=13, multiscale=True))
    model = _model(precision, num_samples=samples)
    full = model(rays, False, True)
    for i in range(b):
        one = model(mp.Rays(*[f[i:i + 1] for f in rays]), False, True)
        for lvl in range(2):
            for k in range(len(full[lvl])):
                if full[lvl][k] is None:
                    continue
                assert torch.equal(one[lvl][k], full[lvl][k][i:i + 1]), (precision, samples, b, i, lvl, k)


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
@pytest.mark.parametrize("mode", ["density", "radiance"])
def test_queries_match_single_tile_launches(precision, mode):
    n = 128 * (_sms() + 1) + 37  # the last tile is part-filled; CTA 0 takes two tiles
    g = torch.Generator().manual_seed(17)
    means = (3.0 * torch.rand(n, 3, generator=g) - 1.5).to(DEV)
    covs = (10 ** (-6 + 5 * torch.rand(n, 3, generator=g))).to(DEV)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV)
    model = _model(precision)

    def query(sl):
        if mode == "density":
            return (model.query_density(means[sl], covs[sl], raw=True),)
        return model.query_radiance(means[sl], covs[sl], dirs[sl], raw=True)

    full = query(slice(0, n))
    for t0 in range(0, n, 128):
        one = query(slice(t0, t0 + 128))
        for a, b in zip(one, full):
            assert torch.equal(a, b[t0:t0 + 128]), (precision, mode, t0)
