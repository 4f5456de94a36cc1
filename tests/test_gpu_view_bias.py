"""The level kernel's per-ray view bias lives in one of two shared-memory slots per CTA (the parity of the ray's index in
the CTA), filled by the helper warps in the ray prologue and read by the view layer's epilogue.  A slot reused too early
would give a ray its neighbour's view bias.  With distinct random view directions per ray, a batch in which every CTA
walks many rays must equal, bit for bit, the same rays rendered in slices of at most one ray per SM, where each CTA
takes a single ray and no slot is reused."""
import pytest
import torch

from helpers import make_state_dict

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"


def _random_viewdirs(rays, seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(rays.viewdirs.shape, generator=g), dim=-1)
    return rays._replace(viewdirs=d)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("n", [128, 256])
@pytest.mark.parametrize("precision", ["bf16", "fp16x3"])
def test_forward_equals_one_ray_per_cta_slices(precision, n):
    b = 4096
    rays = _random_viewdirs(mp.random_ray_batch(b, seed=11, multiscale=True), seed=12)
    rays = mp.namedtuple_map(lambda t: t.to(DEV), rays)
    model = mp.MipNerf(precision=precision, num_samples=n)
    model.load_state_dict(make_state_dict(seed=7, kind="trained_like"))
    model = model.to(DEV).eval()
    whole = model(rays, False, True)
    step = _sms()
    parts = [model(mp.Rays(*[f[i:i + step] for f in rays]), False, True) for i in range(0, b, step)]
    torch.cuda.synchronize()
    for lvl in range(2):
        for k in range(5):
            sliced = torch.cat([p[lvl][k] for p in parts])
            assert torch.equal(whole[lvl][k], sliced), (precision, n, lvl, k)


@pytest.mark.parametrize("precision", ["bf16", "fp16x3"])
def test_mlp_only_mode_equals_one_ray_per_cta_slices(precision):
    b = 2048
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(b, 128, 96, generator=g) * 2 - 1).to(DEV)
    venc = torch.randn(b, 27, generator=g).to(DEV)
    params = make_state_dict(seed=7, kind="trained_like")
    mlp = mp.MLP(8, 256, 1, 128, 4, 3, 1, "relu", 96, 27)
    mlp.load_state_dict({k[len("mlp."):]: v for k, v in params.items()})
    mlp = mlp.to(DEV).eval()
    rgb, dens = mlp(x, venc, precision=precision)
    step = _sms()
    parts = [mlp(x[i:i + step], venc[i:i + step], precision=precision) for i in range(0, b, step)]
    torch.cuda.synchronize()
    assert torch.equal(rgb, torch.cat([p[0] for p in parts]))
    assert torch.equal(dens, torch.cat([p[1] for p in parts]))
