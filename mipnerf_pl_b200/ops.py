"""Host-side mirror of the reference's ray-math free functions (models/mip.py).

Same names, argument meaning and error behaviour as the reference; each call
marshals CUDA tensors into the matching C-ABI entry point of
libmipnerf_b200.so.  CPU tensors are rejected: there is no fallback path.

Differences that the C ABI forces and that are visible here:
  * random draws are explicit optional arguments (`t_rand`, `u_jitter`, `density_normal`) so a
    caller (or a parity test) can inject the noise; when omitted they are
    drawn with torch's CUDA generator;
  * everything is fp32; other dtypes are cast at the boundary.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
from torch.autograd.function import once_differentiable

from . import _cabi

F32_EPS = float(torch.finfo(torch.float32).eps)


def _dev(t: torch.Tensor) -> torch.device:
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise RuntimeError("mipnerf_pl_b200 runs on CUDA tensors only (no CPU fallback); "
                           f"got {getattr(t, 'device', type(t))}")
    return t.device


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(dtype=torch.float32).contiguous()


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _call(dev: torch.device, what: str, fn, *args) -> None:
    """Launch the library entry point `fn(*args, stream)` on `dev`'s current stream, the last argument of every entry
    point that launches, and raise its error as `_cabi.check` does.  The device is made current only when it is not
    already: the guard costs host time on every call."""
    if dev.index is not None and dev.index != torch.cuda.current_device():
        with torch.cuda.device(dev):
            return _call(dev, what, fn, *args)
    _cabi.check(fn(*args, _stream(dev)), what)


def _rays_struct(origins, directions, viewdirs, radii, near=None, far=None):
    """(RaysStruct, keep): `keep` holds the fp32 ray tensors the struct points at, in its field order; viewdirs may be
    None (NULL), near / far default to zeros."""
    n = origins.shape[0]
    zeros = lambda: torch.zeros(n, device=origins.device)  # noqa: E731
    keep = [_f32(origins), _f32(directions), _f32(viewdirs) if viewdirs is not None else None, _f32(radii).reshape(-1),
            _f32(near).reshape(-1) if near is not None else zeros(), _f32(far).reshape(-1) if far is not None else zeros()]
    return _cabi.RaysStruct(*[_ptr(k) for k in keep], n), keep


def _grad_array(grads):
    """The LinearGrad array over (weight, bias) gradient tensors in `MLP.linears()` order."""
    arr = (_cabi.LinearGrad * (len(grads) // 2))()
    for i in range(len(arr)):
        arr[i] = _cabi.LinearGrad(grads[2 * i].data_ptr(), grads[2 * i + 1].data_ptr())
    return arr


def draw_t_rand(batch: int, num_samples: int, device) -> torch.Tensor:
    """torch.rand(batch, N+1) of models/mip.py:159."""
    return torch.rand(batch, num_samples + 1, device=device, dtype=torch.float32)


def draw_u_jitter(batch: int, num_draws: int, device) -> torch.Tensor:
    """uniform_(to=1/num_draws - eps) of models/mip.py:201-202."""
    return torch.empty(batch, num_draws, device=device, dtype=torch.float32).uniform_(
        0.0, 1.0 / num_draws - F32_EPS)


def philox_uniform(seed: int, offset: int, stream_id: int, batch: int, num_draws: int, device) -> torch.Tensor:
    """The uniforms the kernels draw in-kernel for (seed, offset): stream 0 = t_rand in [0,1) (models/mip.py:159),
    stream 1 + level = that level's u_jitter in [0, 1/num_draws - eps) (models/mip.py:201-202).  Passing them as
    `t_rand` / `u_jitter` reproduces the in-kernel randomized forward bit for bit."""
    dev = torch.device(device)
    out = torch.empty(batch, num_draws, device=dev)
    rng = _cabi.Rng(seed & 0xFFFFFFFFFFFFFFFF, offset)
    _call(dev, "philox_uniform", _cabi.lib().mipnerf_b200_philox_uniform, C.byref(rng), stream_id, batch, num_draws,
          out.data_ptr())
    return out


def draw_density_normal(batch: int, num_samples: int, device) -> torch.Tensor:
    """torch.randn(raw_density.shape) of models/mip_nerf.py:233 (one [B,N] draw per level)."""
    return torch.randn(batch, num_samples, device=device, dtype=torch.float32)


def philox_normal(seed: int, offset: int, level: int, batch: int, num_samples: int, device) -> torch.Tensor:
    """The standard normals the kernels draw in-kernel for (seed, offset) as the density noise of `level`
    (models/mip_nerf.py:232-233).  Passed as `density_normal[level]` they reproduce the in-kernel randomized
    forward bit for bit."""
    dev = torch.device(device)
    out = torch.empty(batch, num_samples, device=dev)
    rng = _cabi.Rng(seed & 0xFFFFFFFFFFFFFFFF, offset)
    _call(dev, "philox_normal", _cabi.lib().mipnerf_b200_philox_normal, C.byref(rng), level, batch, num_samples,
          out.data_ptr())
    return out


def cast_rays(t_samples, origins, directions, radii, ray_shape, diagonal=True):
    """models/mip.py:81-103."""
    if ray_shape == "cylinder":
        raise NotImplementedError
    assert ray_shape == "cone"
    if not diagonal:
        raise NotImplementedError("full-covariance branch is dead code in the reference (SURVEY §2)")
    dev = _dev(t_samples)
    t = _f32(t_samples)
    b, n = t.shape[0], t.shape[1] - 1
    rs, keep = _rays_struct(origins, directions, None, radii)
    means = torch.empty(b, n, 3, device=dev)
    covs = torch.empty(b, n, 3, device=dev)
    _call(dev, "cast_rays", _cabi.lib().mipnerf_b200_cast_rays, C.byref(rs), t.data_ptr(), n, means.data_ptr(),
          covs.data_ptr())
    return means, covs


def sample_along_rays(origins, directions, radii, num_samples, near, far, randomized, disparity, ray_shape,
                      t_rand: Optional[torch.Tensor] = None):
    """models/mip.py:127-165 -> (t_samples [B,N+1], (means, covs))."""
    if ray_shape == "cylinder":
        raise NotImplementedError
    assert ray_shape == "cone"
    dev = _dev(origins)
    b = origins.shape[0]
    rs, keep = _rays_struct(origins, directions, None, radii, near, far)
    if randomized and t_rand is None:
        t_rand = draw_t_rand(b, num_samples, dev)
    tr = _f32(t_rand) if randomized else None
    t = torch.empty(b, num_samples + 1, device=dev)
    means = torch.empty(b, num_samples, 3, device=dev)
    covs = torch.empty(b, num_samples, 3, device=dev)
    _call(dev, "sample_along_rays", _cabi.lib().mipnerf_b200_sample_along_rays, C.byref(rs), num_samples,
          int(bool(randomized)), int(bool(disparity)), _ptr(tr), t.data_ptr(), means.data_ptr(), covs.data_ptr())
    return t, (means, covs)


def sorted_piecewise_constant_pdf(bins, weights, num_samples, randomized,
                                  u_jitter: Optional[torch.Tensor] = None, return_inds: bool = False):
    """models/mip.py:168-229.  `weights` is NOT modified (the reference pads it in place).
    weights [B, nb] with nb a multiple of 32 up to 512, num_samples >= 2; other sizes raise NotImplementedError
    (above 544 bins CPU torch sums a row in another order, so the samples would stop being bit-exact)."""
    dev = _dev(bins)
    bn, w = _f32(bins), _f32(weights)
    b, nb = w.shape
    if randomized and u_jitter is None:
        u_jitter = draw_u_jitter(b, num_samples, dev)
    uj = _f32(u_jitter) if randomized else None
    out = torch.empty(b, num_samples, device=dev)
    inds = torch.empty(b, num_samples, device=dev, dtype=torch.int64) if return_inds else None
    _call(dev, "sorted_piecewise_constant_pdf", _cabi.lib().mipnerf_b200_sorted_piecewise_constant_pdf, bn.data_ptr(),
          w.data_ptr(), b, nb, num_samples, int(bool(randomized)), _ptr(uj), out.data_ptr(), _ptr(inds))
    return (out, inds) if return_inds else out


def resample_along_rays(origins, directions, radii, t_samples, weights, randomized, ray_shape, stop_grad,
                        resample_padding, u_jitter: Optional[torch.Tensor] = None, return_inds: bool = False):
    """models/mip.py:232-280 -> (new_t [B,N+1], (means, covs)).  Forward only, so `stop_grad`
    (which only changes autograd in the reference) has no effect on the values.  weights [B, N] with N a multiple
    of 32 up to 512; other sizes raise NotImplementedError, as in sorted_piecewise_constant_pdf."""
    if ray_shape == "cylinder":
        raise NotImplementedError
    assert ray_shape == "cone"
    dev = _dev(t_samples)
    t, w = _f32(t_samples), _f32(weights)
    b, n = w.shape
    rs, keep = _rays_struct(origins, directions, None, radii)
    if randomized and u_jitter is None:
        u_jitter = draw_u_jitter(b, n + 1, dev)
    uj = _f32(u_jitter) if randomized else None
    new_t = torch.empty(b, n + 1, device=dev)
    means = torch.empty(b, n, 3, device=dev)
    covs = torch.empty(b, n, 3, device=dev)
    inds = torch.empty(b, n + 1, device=dev, dtype=torch.int64) if return_inds else None
    _call(dev, "resample_along_rays", _cabi.lib().mipnerf_b200_resample_along_rays, C.byref(rs), t.data_ptr(),
          w.data_ptr(), n, int(bool(randomized)), _ptr(uj), float(resample_padding), new_t.data_ptr(), means.data_ptr(),
          covs.data_ptr(), _ptr(inds))
    return (new_t, (means, covs), inds) if return_inds else (new_t, (means, covs))


def integrated_pos_enc(means_covs, min_deg, max_deg, diagonal=True):
    """models/mip.py:322-350 (diagonal): ([..,3],[..,3]) -> [.., 6*(max-min)]."""
    if not diagonal:
        raise NotImplementedError("full-covariance branch is dead code in the reference (SURVEY §2)")
    means, covs = means_covs
    dev = _dev(means)
    m, c = _f32(means), _f32(covs)
    lead = m.shape[:-1]
    npts = m.numel() // 3
    out = torch.empty(*lead, 6 * (max_deg - min_deg), device=dev)
    _call(dev, "integrated_pos_enc", _cabi.lib().mipnerf_b200_integrated_pos_enc, m.data_ptr(), c.data_ptr(), npts,
          int(min_deg), int(max_deg), out.data_ptr())
    return out


def pos_enc(x, min_deg, max_deg, append_identity=True):
    """models/mip.py:353-363."""
    dev = _dev(x)
    xx = _f32(x)
    lead = xx.shape[:-1]
    width = 6 * (max_deg - min_deg) + (3 if append_identity else 0)
    out = torch.empty(*lead, width, device=dev)
    _call(dev, "pos_enc", _cabi.lib().mipnerf_b200_pos_enc, xx.data_ptr(), xx.numel() // 3, int(min_deg),
          int(max_deg), int(bool(append_identity)), out.data_ptr())
    return out


def volumetric_rendering(rgb, density, t_samples, dirs, white_bkgd):
    """models/mip.py:366-401 -> (comp_rgb [B,3], distance [B], acc [B], weights [B,N]).
    N in {32, 64, 96, 128, 192, 256}, the forward's sample counts; any other N raises NotImplementedError."""
    dev = _dev(rgb)
    r, d, t, dd = _f32(rgb), _f32(density), _f32(t_samples), _f32(dirs)
    b, n = r.shape[0], r.shape[1]
    comp = torch.empty(b, 3, device=dev)
    dist = torch.empty(b, device=dev)
    acc = torch.empty(b, device=dev)
    w = torch.empty(b, n, device=dev)
    _call(dev, "volumetric_rendering", _cabi.lib().mipnerf_b200_volumetric_rendering, r.data_ptr(), d.data_ptr(),
          t.data_ptr(), dd.data_ptr(), b, n, int(bool(white_bkgd)), comp.data_ptr(), dist.data_ptr(), acc.data_ptr(),
          w.data_ptr())
    return comp, dist, acc, w


def _distloss_value(w: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    dev = _dev(w)
    b, n = w.shape
    out = torch.empty(b, device=dev)
    _call(dev, "distloss", _cabi.lib().mipnerf_b200_distloss, w.data_ptr(), t.data_ptr(), b, n, out.data_ptr())
    return out.mean()


class _DistLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weight, samples):
        w, t = _f32(weight), _f32(samples)
        ctx.save_for_backward(w, t)
        ctx.weight_dtype = weight.dtype
        return _distloss_value(w, t)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        w, t = ctx.saved_tensors
        b, n = w.shape
        dev = w.device
        d_w = torch.empty_like(w)
        g = _f32(grad_out).reshape(1)
        _call(dev, "distloss_backward", _cabi.lib().mipnerf_b200_distloss_backward, w.data_ptr(), t.data_ptr(), b, n,
              g.data_ptr(), 1.0 / max(b, 1), d_w.data_ptr())
        return d_w.to(ctx.weight_dtype), None


def distloss(weight, samples):
    """Distortion loss (models/mip.py:8-20): weight [B,N], samples [B,N+1] -> scalar; O(N) per ray instead of the
    reference's two [B,N,N] temporaries.  Differentiable with respect to `weight` when it requires grad (the
    gradient is the same prefix-sum form, `mipnerf_b200_distloss_backward`); `samples` is a constant, as under
    stop_resample_grad.  Inside `train.forward_backward` the gradient is part of the fused step."""
    _dev(weight)
    if torch.is_grad_enabled() and weight.requires_grad:
        return _DistLoss.apply(weight, samples)
    return _distloss_value(_f32(weight), _f32(samples))


def _interlevel_check(t, w, t_hat, w_hat):
    """interlevel_loss's shape and device refusals."""
    shapes = [tuple(x.shape) for x in (t, w, t_hat, w_hat)]
    if not (all(len(s) == 2 for s in shapes) and len({s[0] for s in shapes}) == 1 and shapes[1][1] >= 1
            and shapes[0][1] == shapes[1][1] + 1 and shapes[3][1] >= 1 and shapes[2][1] == shapes[3][1] + 1):
        raise ValueError(f"interlevel_loss: t {shapes[0]}, w {shapes[1]}, t_hat {shapes[2]}, w_hat {shapes[3]}: need "
                         "[B, N+1], [B, N], [B, M+1], [B, M] with N, M >= 1")
    devs = {x.device for x in (t, w, t_hat, w_hat)}
    if len(devs) != 1:
        raise ValueError(f"interlevel_loss: tensors on {sorted(str(d) for d in devs)}; need one device")


def _interlevel_value(t, w, t_hat, w_hat) -> torch.Tensor:
    dev = _dev(w)
    b, n = w.shape
    out = torch.empty(b, device=dev)
    _call(dev, "interlevel_loss", _cabi.lib().mipnerf_b200_interlevel_loss, t.data_ptr(), w.data_ptr(), n,
          t_hat.data_ptr(), w_hat.data_ptr(), w_hat.shape[1], b, out.data_ptr())
    return out.mean()


class _InterlevelLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t, w, t_hat, w_hat):
        args = [_f32(x) for x in (t, w, t_hat, w_hat)]
        ctx.save_for_backward(*args)
        ctx.w_hat_dtype = w_hat.dtype
        return _interlevel_value(*args)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        t, w, t_hat, w_hat = ctx.saved_tensors
        b, n = w.shape
        d_w_hat = torch.empty_like(w_hat)
        g = _f32(grad_out).reshape(1)
        _call(w.device, "interlevel_loss_backward", _cabi.lib().mipnerf_b200_interlevel_loss_backward, t.data_ptr(),
              w.data_ptr(), n, t_hat.data_ptr(), w_hat.data_ptr(), w_hat.shape[1], b, g.data_ptr(), 1.0 / max(b, 1),
              d_w_hat.data_ptr())
        return None, None, None, d_w_hat.to(ctx.w_hat_dtype)


def interlevel_loss(t, w, t_hat, w_hat):
    """mip-NeRF 360's interlevel loss, the mean over rays of sum_i max(0, w_i - bound_i)^2 / (w_i + eps): fine
    fenceposts t [B,N+1] and weights w [B,N], proposal fenceposts t_hat [B,M+1] and weights w_hat [B,M], bound_i the
    proposal weight of the proposal intervals that overlap fine interval i (`mipnerf_b200_interlevel_loss`).  It
    penalises fine weight the proposal does not cover.  Differentiable with respect to `w_hat` when it requires grad
    (`mipnerf_b200_interlevel_loss_backward`); t, w and t_hat are constants, the paper's stop-gradient.  Deterministic:
    the value and the gradient are bit for bit the same across runs."""
    _interlevel_check(t, w, t_hat, w_hat)
    _dev(w)
    if torch.is_grad_enabled() and w_hat.requires_grad:
        return _InterlevelLoss.apply(t, w, t_hat, w_hat)
    return _interlevel_value(*[_f32(x) for x in (t, w, t_hat, w_hat)])
