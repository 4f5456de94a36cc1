"""The level kernel runs each CTA's rays as a pipeline: the helper warps prepare the next ray's fenceposts and features
in one of the feature buffers and composite the previous ray while the wgmma warpgroups run the layers of the current
one.  A batch of 2 * SMs + 5 rays gives some CTAs three rays and the others two, so every hand-off between rays (feature
buffer parity, raw-heads parity, their waits) is exercised; it must render exactly what single-ray launches render,
which have no neighbouring ray to overlap with."""
import pytest
import torch

from helpers import make_state_dict

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"


def _batch_size():
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count + 5


@pytest.mark.parametrize("randomized", [False, True])
@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp16x3"])
def test_level_pipeline_matches_single_ray_launches(precision, randomized):
    b = _batch_size()
    rays = mp.namedtuple_map(lambda t: t.to(DEV), mp.random_ray_batch(b, seed=41, multiscale=True))
    model = mp.MipNerf(precision=precision, density_noise=1.0)
    model.load_state_dict(make_state_dict(seed=7, kind="trained_like"))
    model = model.to(DEV).eval()
    noise = {}
    if randomized:  # Philox draws from torch's generator, row-sliced below so that every ray sees the same draws
        g = torch.Generator(device=DEV).manual_seed(5)
        noise = dict(t_rand=torch.rand(b, 129, device=DEV, generator=g),
                     u_jitter=torch.rand(b, 129, device=DEV, generator=g) * (1 / 129 - 1.2e-7),
                     density_normal=[torch.randn(b, 128, device=DEV, generator=g) for _ in range(2)])
    full = model(rays, randomized, True, return_inds=True, **noise)
    for i in range(b):
        one_noise = {}
        if randomized:
            one_noise = dict(t_rand=noise["t_rand"][i:i + 1], u_jitter=noise["u_jitter"][i:i + 1],
                             density_normal=[x[i:i + 1] for x in noise["density_normal"]])
        one = model(mp.Rays(*[f[i:i + 1] for f in rays]), randomized, True, return_inds=True, **one_noise)
        for lvl in range(2):
            for k in range(6):
                if full[lvl][k] is None:
                    continue
                assert torch.equal(one[lvl][k], full[lvl][k][i:i + 1]), (precision, i, lvl, k)


@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp16x3"])
def test_level_pipeline_mlp_only_matches_single_ray_launches(precision):
    b = _batch_size()
    g = torch.Generator().manual_seed(43)
    x = (torch.rand(b, 128, 96, generator=g) * 2 - 1).to(DEV)
    venc = torch.randn(b, 27, generator=g).to(DEV)
    params = make_state_dict(seed=6, kind="xavier")
    mlp = mp.MLP(8, 256, 1, 128, 4, 3, 1, "relu", 96, 27)
    mlp.load_state_dict({k[len("mlp."):]: v for k, v in params.items()})
    mlp = mlp.to(DEV).eval()
    rgb, dens = mlp(x, venc, precision=precision)
    for i in range(b):
        rgb1, dens1 = mlp(x[i:i + 1], venc[i:i + 1], precision=precision)
        assert torch.equal(rgb1, rgb[i:i + 1]) and torch.equal(dens1, dens[i:i + 1]), (precision, i)
