"""`MLP` and `MipNerf` with the reference's constructor signatures, submodule
tree and state_dict keys (models/mip_nerf.py:14-248), whose `forward` runs on
the sm_90a kernels of libmipnerf_b200.so through the C ABI.

The modules own ordinary fp32 `torch.nn.Linear` parameters, so Lightning
checkpoints of the reference (`mip_nerf.mlp.layers.{i}.0.weight`, ...) load with
`load_state_dict` unchanged.

Training, two ways:
  * `mipnerf_pl_b200.train` (`fused_loss` / `forward_backward`): one library call runs forward and backward of the
    reference's loss (masked MSE per level + 0.01 distloss, coarse multiplier) and hands the gradients to autograd
    or `param.grad`.  The fastest step, but the loss is fixed.
  * `MipNerf(autograd=True)`: `forward` returns outputs with a `grad_fn` over the 24 MLP tensors (when grad mode is
    on and a parameter requires grad), so any loss on comp_rgb / distance / acc / weights trains through
    `loss.backward()`.  Only the rays, the fenceposts and the density noise are kept between the two passes
    (O(B*N) floats, no activations); the backward re-runs the training forward at those fenceposts chunk by chunk
    and then the library's backward chain (`mipnerf_b200_backward`).  fp32 and bf16; t_samples carry no gradient
    (stop_resample_grad=True).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import torch
from torch.autograd.function import once_differentiable

from . import _cabi
from .ops import _call, _dev, _f32, _grad_array, _ptr, _rays_struct, draw_density_normal, draw_t_rand, draw_u_jitter
from .rays import Rays


def _xavier_init(linear):
    torch.nn.init.xavier_uniform_(linear.weight.data)


class _Workspace:
    """Per-(device, stream) scratch handed to the library (torch owns every byte, SURVEY §8b).  Keyed by the stream
    the call is enqueued on, so forwards issued on different streams never share a scratch buffer."""
    _bufs = {}

    @classmethod
    def get(cls, device: torch.device, nbytes: int) -> torch.Tensor:
        key = (device.type, device.index if device.index is not None else torch.cuda.current_device(),
               torch.cuda.current_stream(device).cuda_stream)
        buf = cls._bufs.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = None
            cls._bufs.pop(key, None)
            buf = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=device)
            cls._bufs[key] = buf
        return buf


class MLP(torch.nn.Module):
    """models/mip_nerf.py:14-111 — same constructor, same parameter names."""

    def __init__(self, net_depth: int, net_width: int, net_depth_condition: int, net_width_condition: int,
                 skip_index: int, num_rgb_channels: int, num_density_channels: int, activation: str,
                 xyz_dim: int, view_dim: int):
        super().__init__()
        if activation != "relu":
            raise NotImplementedError  # models/mip_nerf.py:49-50
        self.net_depth, self.net_width = net_depth, net_width
        self.net_depth_condition, self.net_width_condition = net_depth_condition, net_width_condition
        self.skip_index = skip_index
        self.num_rgb_channels, self.num_density_channels = num_rgb_channels, num_density_channels
        self.xyz_dim, self.view_dim = xyz_dim, view_dim
        layers = []
        for i in range(net_depth):
            if i == 0:
                dim_in = xyz_dim
            elif (i - 1) % skip_index == 0 and i > 1:
                dim_in = net_width + xyz_dim
            else:
                dim_in = net_width
            linear = torch.nn.Linear(dim_in, net_width)
            _xavier_init(linear)
            layers.append(torch.nn.Sequential(linear, torch.nn.ReLU(True)))
        self.layers = torch.nn.ModuleList(layers)
        self.density_layer = torch.nn.Linear(net_width, num_density_channels)
        _xavier_init(self.density_layer)
        self.extra_layer = torch.nn.Linear(net_width, net_width)
        _xavier_init(self.extra_layer)
        layers = []
        for i in range(net_depth_condition):
            dim_in = net_width + view_dim if i == 0 else net_width_condition
            linear = torch.nn.Linear(dim_in, net_width_condition)
            _xavier_init(linear)
            layers.append(torch.nn.Sequential(linear, torch.nn.ReLU(True)))
        self.view_layers = torch.nn.Sequential(*layers)
        self.color_layer = torch.nn.Linear(net_width_condition, num_rgb_channels)

    def __getstate__(self):  # ctypes marshalling caches are per-process
        d = self.__dict__.copy()
        d.pop("_ws_cache", None)
        d.pop("_lin_cache", None)
        return d

    # ---- marshalling --------------------------------------------------------------------------
    def linears(self) -> List[torch.nn.Linear]:
        """state_dict order expected by mipnerf_b200_weights (cached: the submodule tree is fixed after __init__)."""
        lins = self.__dict__.get("_lin_cache")
        if lins is None:
            lins = ([seq[0] for seq in self.layers] + [self.density_layer, self.extra_layer] +
                    [seq[0] for seq in self.view_layers] + [self.color_layer])
            self.__dict__["_lin_cache"] = lins
        return lins

    def params(self) -> List[torch.nn.Parameter]:
        """weight, bias of every layer in `linears()` order: the order of the library's gradient arrays."""
        return [p for lin in self.linears() for p in (lin.weight, lin.bias)]

    def _weights_struct(self, cfg: "_cabi.Config", precision: int, device):
        """(struct, keep-alive list) for `precision` on `device`.  Cached per (precision, device) until a parameter is
        modified, moved or re-typed; every precision's struct points at the same fp32 parameter tensors, and a
        tensor-core precision adds its packed weight image."""
        lins = self.linears()
        state = tuple((l.weight.data_ptr(), l.weight._version, l.bias.data_ptr(), l.bias._version, l.weight.dtype)
                      for l in lins)
        cache = self.__dict__.get("_ws_cache")
        if cache is None or cache[0] != state:
            cache = self.__dict__["_ws_cache"] = (state, {})
        key = (precision, str(device))
        hit = cache[1].get(key)
        if hit is not None:
            return hit
        if precision == _cabi.FP32:
            arr = (_cabi.Linear * len(lins))()
            keep = []
            for i, l in enumerate(lins):
                w, b = _f32(l.weight), _f32(l.bias)
                if w.device != device:
                    raise RuntimeError(f"MLP parameters live on {w.device}, rays on {device}")
                keep += [w, b]
                arr[i] = _cabi.Linear(w.data_ptr(), b.data_ptr(), l.in_features, l.out_features)
            hit = (_cabi.Weights(arr, len(lins), -1, None, 0), keep + [arr])
        else:
            ws, keep = self._weights_struct(cfg, _cabi.FP32, device)
            hit = self._packed_image(cfg, ws, precision, device, keep)
        cache[1][key] = hit
        return hit

    def _packed_image(self, cfg, ws, precision, device, keep):
        """(struct, keep-alive list) of a tensor-core precision: the fp32 struct `ws` (whose tensors `keep` holds) plus
        its weight image, packed on `device`."""
        lib = _cabi.lib()
        nbytes = lib.mipnerf_b200_packed_weights_bytes(C.byref(cfg), precision)
        if nbytes == 0:
            raise NotImplementedError("tensor-core path: the 8x256 / 1x128 MLP with num_samples 128 or 256, "
                                      "min_deg_point=0, max_deg_point 1..16 and deg_view 1..4 is implemented; "
                                      "use precision='fp32'")
        packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _call(device, "pack_weights", lib.mipnerf_b200_pack_weights, C.byref(cfg), C.byref(ws), precision,
              packed.data_ptr(), nbytes)
        return (_cabi.Weights(ws.linears, ws.num_linears, precision, packed.data_ptr(), packed.numel()),
                keep + [packed])

    def _config(self, num_samples=128, **over) -> "_cabi.Config":
        deg_pts = self.xyz_dim // 6
        deg_view = (self.view_dim - 3) // 6
        vals = dict(num_samples=num_samples, num_levels=1, min_deg_point=0, max_deg_point=deg_pts,
                    deg_view=deg_view, use_viewdirs=1, disparity=0, disable_integration=0,
                    resample_padding=0.01, density_bias=-1.0, rgb_padding=0.001, net_depth=self.net_depth,
                    net_width=self.net_width, net_depth_condition=self.net_depth_condition,
                    net_width_condition=self.net_width_condition, skip_index=self.skip_index,
                    num_rgb_channels=self.num_rgb_channels, num_density_channels=self.num_density_channels)
        vals.update(over)
        return _cabi.Config(**vals)

    def forward(self, x, view_direction=None, precision: str = "fp32"):
        """models/mip_nerf.py:75-111: x [B,N,xyz_dim], view_direction [B,view_dim] ->
        (raw_rgb [B,N,3], raw_density [B,N,1])."""
        dev = _dev(x)
        xx = _f32(x)
        b, n = xx.shape[0], xx.shape[1]
        vd = _f32(view_direction) if view_direction is not None else None
        prec = _cabi.PRECISIONS[precision]
        cfg = self._config(use_viewdirs=int(vd is not None))
        ws, keep = self._weights_struct(cfg, prec, dev)
        lib = _cabi.lib()
        raw_rgb = torch.empty(b, n, 3, device=dev)
        raw_density = torch.empty(b, n, 1, device=dev)
        nbytes = lib.mipnerf_b200_mlp_workspace_bytes(C.byref(cfg), b, n, prec)
        scratch = _Workspace.get(dev, nbytes)
        _call(dev, "MLP.forward", lib.mipnerf_b200_mlp_forward, C.byref(cfg), C.byref(ws), xx.data_ptr(), _ptr(vd), b,
              n, prec, raw_rgb.data_ptr(), raw_density.data_ptr(), scratch.data_ptr(), scratch.numel())
        return raw_rgb, raw_density


class LevelOutputs(list):
    """What `MipNerf.forward` returns: the reference's list of per-level 5-tuples (models/mip_nerf.py:246), plus
    `.pixels` — comp_rgb | distance | acc of every level as one contiguous [levels, 5*B] tensor (a view of the same
    memory), for reading rendered pixels back to the host with a single copy."""
    pixels: Optional[torch.Tensor] = None


def _level_outputs(b: int, n: int, levels: int, dev, normals, return_inds: bool, first: int = 0):
    """(LevelOutputs, LevelOut array) of a call on b rays with n samples per level, in one allocation: the pixel outputs
    (comp_rgb | distance | acc = 5 floats per ray) of all levels first, so that a caller that only wants pixels reads
    them back with ONE contiguous copy (`.pixels`, [levels, 5*B]); then weights / fenceposts per level.  `normals`: the
    density normals handed to the library, one tensor or None per level.  `first`: the model level of entry 0 (1 for
    `forward_proposed`, whose levels all resample and so all have inds)."""
    flat = torch.empty(levels * b * (5 + n + n + 1), device=dev)
    ret = LevelOutputs()
    ret.pixels = flat[:levels * 5 * b].view(levels, 5 * b) if b > 0 else flat[:0].view(levels, 0)
    outs = (_cabi.LevelOut * levels)()
    tail = levels * 5 * b
    for lvl in range(levels):
        o = lvl * 5 * b
        comp = flat[o:o + 3 * b].view(b, 3)
        dist = flat[o + 3 * b:o + 4 * b]
        acc = flat[o + 4 * b:o + 5 * b]
        q = tail + lvl * (2 * n + 1) * b
        w = flat[q:q + n * b].view(b, n)
        t = flat[q + n * b:q + (2 * n + 1) * b].view(b, n + 1)
        inds = torch.empty(b, n + 1, device=dev, dtype=torch.int64) if (return_inds and lvl + first > 0) else None
        outs[lvl] = _cabi.LevelOut(comp.data_ptr(), dist.data_ptr(), acc.data_ptr(), w.data_ptr(), t.data_ptr(),
                                   _ptr(inds), _ptr(normals[lvl]))
        ret.append((comp, dist, acc, w, t, inds) if return_inds else (comp, dist, acc, w, t))
    return ret, outs


def _shape(x: Optional[torch.Tensor]):
    return None if x is None else tuple(x.shape)


def _query_points(what: str, means: torch.Tensor, covs: Optional[torch.Tensor], viewdirs: Optional[torch.Tensor] = None,
                  dirs: Optional[torch.Tensor] = None, table: Optional[torch.Tensor] = None):
    """Check the arguments of a field query -> (leading shape, means, covs, viewdirs, dirs, table): means / covs /
    viewdirs flattened to fp32 [P, 3], dirs [D, 3] and table [D, K] fp32 on means' device; None stays None.  Only
    shapes are checked: a CPU tensor is refused where it is handed to the library."""
    if means.shape[-1] != 3 or any(x is not None and x.shape != means.shape for x in (covs, viewdirs)):
        raise ValueError(f"{what}: means {_shape(means)} / covs {_shape(covs)} / viewdirs {_shape(viewdirs)}: need "
                         "[..., 3] of the same shape")
    if dirs is not None and (dirs.dim() != 2 or dirs.shape[1] != 3 or dirs.shape[0] < 1):
        raise ValueError(f"{what}: dirs {_shape(dirs)}: need [D, 3] with D >= 1")
    if table is not None and (table.dim() != 2 or table.shape[0] != dirs.shape[0] or not 1 <= table.shape[1] <= 16):
        raise ValueError(f"{what}: table {_shape(table)}: need [D = {dirs.shape[0]}, K] with 1 <= K <= 16")
    return (means.shape[:-1], *[None if x is None else _f32(x).reshape(-1, 3) for x in (means, covs, viewdirs)],
            *[None if x is None else _f32(x).to(means.device) for x in (dirs, table)])


class MipNerf(torch.nn.Module):
    """models/mip_nerf.py:114-248 — same constructor (plus `precision`), same forward contract."""

    def __init__(self, num_samples: int = 128, num_levels: int = 2, resample_padding: float = 0.01,
                 stop_resample_grad: bool = True, use_viewdirs: bool = True, disparity: bool = False,
                 ray_shape: str = 'cone', min_deg_point: int = 0, max_deg_point: int = 16, deg_view: int = 4,
                 density_activation: str = 'softplus', density_noise: float = 0., density_bias: float = -1.,
                 rgb_activation: str = 'sigmoid', rgb_padding: float = 0.001,
                 disable_integration: bool = False, append_identity: bool = True, mlp_net_depth: int = 8,
                 mlp_net_width: int = 256, mlp_net_depth_condition: int = 1, mlp_net_width_condition: int = 128,
                 mlp_skip_index: int = 4, mlp_num_rgb_channels: int = 3, mlp_num_density_channels: int = 1,
                 mlp_net_activation: str = 'relu', precision: Optional[str] = None, autograd: bool = False):
        super().__init__()
        self.num_levels = num_levels
        self.num_samples = num_samples
        self.disparity = disparity
        self.ray_shape = ray_shape
        self.disable_integration = disable_integration
        self.min_deg_point = min_deg_point
        self.max_deg_point = max_deg_point
        self.use_viewdirs = use_viewdirs
        self.deg_view = deg_view
        self.density_noise = density_noise
        self.density_bias = density_bias
        self.resample_padding = resample_padding
        self.stop_resample_grad = stop_resample_grad
        mlp_xyz_dim = (max_deg_point - min_deg_point) * 3 * 2
        mlp_view_dim = deg_view * 3 * 2
        mlp_view_dim = mlp_view_dim + 3 if append_identity else mlp_view_dim
        self.mlp = MLP(mlp_net_depth, mlp_net_width, mlp_net_depth_condition, mlp_net_width_condition,
                       mlp_skip_index, mlp_num_rgb_channels, mlp_num_density_channels, mlp_net_activation,
                       mlp_xyz_dim, mlp_view_dim)
        if rgb_activation != 'sigmoid':
            raise NotImplementedError  # models/mip_nerf.py:162-165
        self.rgb_padding = rgb_padding
        if density_activation != 'softplus':
            raise NotImplementedError  # models/mip_nerf.py:167-170
        # forward() always encodes viewdirs with append_identity=True (models/mip_nerf.py:221-226);
        # a model built with append_identity=False has a 24-wide view input and fails in the reference.
        self._append_identity = bool(append_identity)
        # 'fp32' | 'bf16' | 'fp16' | 'fp16x3' | 'bf16x3'; None -> $MIPNERF_B200_PRECISION or 'fp32'
        self.precision = precision or os.environ.get("MIPNERF_B200_PRECISION", "fp32")
        # randomized=True without injected noise draws its uniforms inside the kernels (Philox4x32-10, counter-based):
        # seed from torch's global generator at first use, offset advanced by one per call.
        self.rng_seed: Optional[int] = None
        self.rng_offset = 0
        # forward builds an autograd graph (grad mode on, some MLP parameter requires grad): any loss on the outputs
        # can call backward(); the gradients come from mipnerf_b200_backward
        self.autograd = bool(autograd)

    def next_rng(self) -> "_cabi.Rng":
        """(seed, offset) of the next randomized call; advances the offset (the role of torch's generator offset)."""
        if self.rng_seed is None:
            self.rng_seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        rng = _cabi.Rng(self.rng_seed, self.rng_offset)
        self.rng_offset += 1
        return rng

    def _noise(self, randomized: bool, b: int, dev, t_rand, u_jitter, density_normal):
        """The noise of a call on b rays -> (rng, t_rand, u_jitter, normals).  randomized without any injected array:
        the kernels draw in-kernel from `next_rng()`.  Otherwise the arrays not given are drawn with torch's generator,
        and `normals` holds one [B,N] tensor per level when density_noise > 0 (models/mip_nerf.py:232-233)."""
        levels, n = self.num_levels, self.num_samples
        if not randomized:
            return None, None, None, [None] * levels
        if t_rand is None and u_jitter is None and density_normal is None:
            return self.next_rng(), None, None, [None] * levels  # no torch.rand launch, no [B,N+1] arrays
        t_rand = _f32(t_rand) if t_rand is not None else draw_t_rand(b, n, dev)
        u_jitter = _f32(u_jitter) if u_jitter is not None else draw_u_jitter(b, n + 1, dev)
        normals = list(density_normal) if density_normal is not None else [None] * levels
        if len(normals) != levels:
            raise ValueError(f"density_normal: expected {levels} tensors (one per level)")
        if not self.density_noise > 0:
            return None, t_rand, u_jitter, [None] * levels
        return None, t_rand, u_jitter, [_f32(x).reshape(b, n) if x is not None else draw_density_normal(b, n, dev)
                                        for x in normals]

    def _config(self) -> "_cabi.Config":
        return self.mlp._config(
            num_samples=self.num_samples, num_levels=self.num_levels, min_deg_point=self.min_deg_point,
            max_deg_point=self.max_deg_point, deg_view=self.deg_view, use_viewdirs=int(bool(self.use_viewdirs)),
            disparity=int(bool(self.disparity)), disable_integration=int(bool(self.disable_integration)),
            resample_padding=float(self.resample_padding), density_bias=float(self.density_bias),
            rgb_padding=float(self.rgb_padding), density_noise=float(self.density_noise))

    def forward(self, rays: Rays, randomized: bool, white_bkgd: bool, *, t_rand: Optional[torch.Tensor] = None,
                u_jitter: Optional[torch.Tensor] = None, density_normal=None, return_inds: bool = False):
        """rays -> [(comp_rgb [B,3], distance [B], acc [B], weights [B,N], t_samples [B,N+1])] * levels
        (models/mip_nerf.py:172-248).  `t_rand` / `u_jitter` / `density_normal` (one [B,N] tensor of standard normals
        per level, models/mip_nerf.py:233) inject the noise of randomized mode; without any of them the kernels draw
        in-kernel.  With `return_inds` a sixth element (searchsorted indices, None for level 0) is appended.

        With `autograd=True`, grad mode on and a parameter that requires grad, comp_rgb / distance / acc / weights of
        every level carry a `grad_fn` over the MLP tensors (values identical: the same launches run); t_samples and
        inds are constants (stop_resample_grad) and `.pixels` has no grad.  fp32 and bf16 only; ray tensors that
        require grad are refused."""
        if self._builds_graph():
            return _forward_with_grad(self, rays, randomized, white_bkgd, t_rand, u_jitter, density_normal, return_inds)
        return self._forward(rays, randomized, white_bkgd, t_rand, u_jitter, density_normal, return_inds)[0]

    @torch.no_grad()
    def forward_proposed(self, rays: Rays, grid, randomized: bool, white_bkgd: bool, *,
                         t_rand: Optional[torch.Tensor] = None, u_jitter: Optional[torch.Tensor] = None,
                         density_normal=None, return_inds: bool = False):
        """`forward` with level 0's MLP replaced by a baked grid's proposal (mip-NeRF 360's proposal sampling) ->
        levels 1..L-1 of `forward`'s list, in its tuple format.  Level 0's fenceposts are the library's
        `sample_along_rays` (t_rand, or Philox stream 0 of `next_rng()` when randomized with no draws given), its
        weights `grid.proposal(rays, t_samples)` (`BakedGrid.proposal`); the later levels resample from those on the
        unchanged level kernels, with `forward`'s draws (u_jitter; density_normal is one tensor per level as for
        `forward`, level 0's unused).  Inference only: no graph, also on an autograd model."""
        t0, rng, u_jitter, normals = self._proposal_fenceposts(rays, randomized, t_rand, u_jitter, density_normal)
        return self._forward_from(rays, t0, grid.proposal(rays, t0), randomized, white_bkgd, rng, u_jitter, normals,
                                  return_inds)

    def _check_proposed(self, what: str) -> None:
        """The refusals of a model whose level 0 a proposal replaces (`forward_proposed`, `finetune_proposal`)."""
        if self.num_levels < 2:
            raise ValueError(f"{what}: num_levels={self.num_levels}; the proposal replaces level 0 of a "
                             "model with at least 2 levels")
        if self.ray_shape != 'cone':
            raise NotImplementedError(f"{what}: ray_shape={self.ray_shape!r}")  # models/mip.py:97-98
        if self.use_viewdirs and not self._append_identity:
            raise RuntimeError("append_identity=False: view encoding width does not match view_layers "
                               "(same failure as the reference)")

    def _proposal_fenceposts(self, rays: Rays, randomized: bool, t_rand, u_jitter, density_normal):
        """Level 0's fenceposts of a forward whose level 0 a proposal replaces -> (t0 [B,N+1], rng, u_jitter, normals):
        the library's `sample_along_rays` with t_rand, or Philox stream 0 of `next_rng()` when randomized with no
        draws given; the rest as `_noise` returns them, for `_forward_from`."""
        self._check_proposed("forward_proposed")
        dev = _dev(rays.origins)
        b, n = rays.origins.shape[0], self.num_samples
        rs, keep = _rays_struct(rays.origins, rays.directions, rays.viewdirs, rays.radii, rays.near, rays.far)
        rng, t_rand, u_jitter, normals = self._noise(randomized, b, dev, t_rand, u_jitter, density_normal)
        lib = _cabi.lib()
        t0 = torch.empty(b, n + 1, device=dev)
        if rng is not None:
            t_rand = torch.empty(b, n + 1, device=dev)
            _call(dev, "philox_uniform", lib.mipnerf_b200_philox_uniform, C.byref(rng), 0, b, n + 1, t_rand.data_ptr())
        _call(dev, "sample_along_rays", lib.mipnerf_b200_sample_along_rays, C.byref(rs), n, int(bool(randomized)),
              int(bool(self.disparity)), _ptr(t_rand), t0.data_ptr(), None, None)
        return t0, rng, u_jitter, normals

    def _forward_from(self, rays: Rays, t_prev: torch.Tensor, w_prev: torch.Tensor, randomized: bool,
                      white_bkgd: bool, rng, u_jitter, normals, return_inds: bool):
        """Levels 1..L-1 of `forward` from level-0 fenceposts t_prev [B,N+1] and weights w_prev [B,N]
        (mipnerf_b200_forward_proposed(_rng)); rng / u_jitter / normals as `_noise` returns them."""
        dev = _dev(rays.origins)
        b, n = rays.origins.shape[0], self.num_samples
        prec = _cabi.PRECISIONS[self.precision]
        cfg = self._config()
        rs, keep = _rays_struct(rays.origins, rays.directions, rays.viewdirs, rays.radii, rays.near, rays.far)
        t_prev, w_prev = _f32(t_prev), _f32(w_prev)
        if tuple(t_prev.shape) != (b, n + 1) or tuple(w_prev.shape) != (b, n):
            raise ValueError(f"t_prev {tuple(t_prev.shape)} / w_prev {tuple(w_prev.shape)}: need [{b}, {n + 1}] / "
                             f"[{b}, {n}]")
        ws, wkeep = self.mlp._weights_struct(cfg, prec, dev)
        ret, outs = _level_outputs(b, n, self.num_levels - 1, dev, normals[1:], return_inds, first=1)
        lib = _cabi.lib()
        scratch = _Workspace.get(dev, lib.mipnerf_b200_workspace_bytes(C.byref(cfg), b, prec))
        args = (C.byref(cfg), C.byref(ws), C.byref(rs), t_prev.data_ptr(), w_prev.data_ptr())
        if rng is not None:
            _call(dev, "MipNerf.forward_proposed", lib.mipnerf_b200_forward_proposed_rng, *args, C.byref(rng),
                  int(bool(white_bkgd)), prec, outs, scratch.data_ptr(), scratch.numel())
        else:
            _call(dev, "MipNerf.forward_proposed", lib.mipnerf_b200_forward_proposed, *args, int(bool(randomized)),
                  _ptr(u_jitter), int(bool(white_bkgd)), prec, outs, scratch.data_ptr(), scratch.numel())
        return ret

    def _builds_graph(self) -> bool:
        """`forward` and the queries return outputs with a grad_fn: autograd=True, grad mode on, and some MLP
        parameter that requires grad."""
        return self.autograd and torch.is_grad_enabled() and any(p.requires_grad for p in self.mlp.parameters())

    def query_density(self, means: torch.Tensor, covs: Optional[torch.Tensor] = None, *, raw: bool = False):
        """Density of the field at Gaussians: means / diagonal covs [..., 3] (covs None: zero covariance) -> [...] on
        `self.precision`: the IPE (models/mip.py:322-350), trunk and density_layer of MLP.forward
        (models/mip_nerf.py:93-98), then softplus(raw + density_bias) unless `raw` (no density noise).  The tensor-core
        precisions take the configs `forward` takes on the tensor cores; fp32 any.

        With `autograd=True`, grad mode on and a parameter that requires grad, the result carries a `grad_fn` over the
        24 MLP tensors (same values: the same launches run); its backward is `mipnerf_b200_query_backward`.  fp32 and
        bf16 (default encodings) only; means / covs that require grad are refused.  Otherwise no grad_fn."""
        shape, m, c = _query_points("query_density", means, covs)[:3]
        if self._builds_graph():
            return _query_with_grad(self, (means, covs), shape, m, c, None, raw)
        with torch.no_grad():
            return self._query_density(m, c, raw).reshape(shape)

    def _query_density(self, m: torch.Tensor, c: Optional[torch.Tensor], raw: bool):
        """The density [P] at the flat fp32 points of `_query_points`."""
        dev = _dev(m)
        p = m.shape[0]
        prec = _cabi.PRECISIONS[self.precision]
        cfg = self._config()
        ws, keep = self.mlp._weights_struct(cfg, prec, dev)
        out = torch.empty(p, device=dev)
        if p == 0:
            return out
        lib = _cabi.lib()
        nbytes = lib.mipnerf_b200_density_workspace_bytes(C.byref(cfg), p, prec)
        scratch = _Workspace.get(dev, nbytes)
        _call(dev, "MipNerf.query_density", lib.mipnerf_b200_query_density, C.byref(cfg), C.byref(ws), m.data_ptr(),
              _ptr(c), p, prec, out.data_ptr() if raw else None, None if raw else out.data_ptr(), scratch.data_ptr(),
              scratch.numel())
        return out

    def query_radiance(self, means: torch.Tensor, covs: Optional[torch.Tensor] = None,
                       viewdirs: Optional[torch.Tensor] = None, *, raw: bool = False):
        """Radiance of the field at Gaussians, each seen from its own direction: means / diagonal covs / viewdirs
        [..., 3] -> (rgb [..., 3], density [...]) on `self.precision`: MLP.forward of the points' IPE features and view
        encodings (models/mip_nerf.py:75-111), then the activations (models/mip_nerf.py:236-237), or the raw heads
        (raw_rgb, raw_density) when `raw`.  No density noise.  viewdirs are encoded as given; the reference encodes
        unit directions.  They may be None only for a model with use_viewdirs=False (fp32: the colour head then reads
        the trunk).  The tensor-core precisions take the configs `forward` takes on the tensor cores (the radiance mode
        of the level kernel); fp32 any.  Gradients with respect to the MLP tensors as for `query_density`."""
        shape, m, c, v = _query_points("query_radiance", means, covs, viewdirs)[:4]
        if viewdirs is None and self.use_viewdirs:
            raise ValueError("query_radiance: viewdirs are required when use_viewdirs=True")
        if self._builds_graph():
            return _query_with_grad(self, (means, covs, viewdirs), shape, m, c, v, raw)
        with torch.no_grad():
            rgb, dens = self._query_radiance(m, c, v, raw)
        return rgb.reshape(*shape, 3), dens.reshape(shape)

    def _query_radiance(self, m: torch.Tensor, c: Optional[torch.Tensor], v: Optional[torch.Tensor], raw: bool):
        """(rgb [P, 3], density [P]) at the flat fp32 points and view directions of `_query_points`."""
        dev = _dev(m)
        p = m.shape[0]
        prec = _cabi.PRECISIONS[self.precision]
        cfg = self._config()
        ws, keep = self.mlp._weights_struct(cfg, prec, dev)
        out_rgb = torch.empty(p, 3, device=dev)
        out_dens = torch.empty(p, device=dev)
        if p > 0:
            lib = _cabi.lib()
            nbytes = lib.mipnerf_b200_radiance_workspace_bytes(C.byref(cfg), p, prec)
            scratch = _Workspace.get(dev, nbytes)
            rgb_ptrs = (out_rgb.data_ptr(), out_dens.data_ptr(), None, None) if raw else \
                (None, None, out_rgb.data_ptr(), out_dens.data_ptr())
            _call(dev, "MipNerf.query_radiance", lib.mipnerf_b200_query_radiance, C.byref(cfg), C.byref(ws),
                  m.data_ptr(), _ptr(c), _ptr(v), p, prec, *rgb_ptrs, scratch.data_ptr(), scratch.numel())
        return out_rgb, out_dens

    def query_radiance_dirs(self, means: torch.Tensor, covs: Optional[torch.Tensor], dirs: torch.Tensor, *,
                            raw: bool = False):
        """Radiance of the field at Gaussians under one shared set of directions: means / diagonal covs [..., 3] (covs
        None: zero covariance), dirs [D, 3] (encoded as given) -> (rgb [..., D, 3], density [...]); `raw`: the raw
        heads instead.  `rgb[..., d, :]` is `query_radiance(means, covs, dirs[d].expand_as(means))[0]` (bit for bit on
        the tensor cores; fp32 to round-off), but the trunk runs once per point and only the view layer's ReLU and the
        colour head once per (point, direction).  Needs use_viewdirs; no autograd (refused where `forward` would build
        a graph)."""
        rgb, dens, _ = self._query_radiance_dirs(means, covs, dirs, None, raw, colors=True)
        return rgb, dens

    def query_radiance_proj(self, means: torch.Tensor, covs: Optional[torch.Tensor], dirs: torch.Tensor,
                            table: torch.Tensor, *, raw: bool = False):
        """The colours of `query_radiance_dirs` projected onto K <= 16 functions of the direction, without forming the
        [..., D, 3] colours: coeffs[..., k, :] = sum over d = 0..D-1 (in order, fp32) of table[d, k] * rgb[..., d, :]
        (raw heads when `raw`) -> (coeffs [..., K, 3], density [...]).  table [D, K], e.g. quadrature weights times a
        basis (`field.bake_sh`).  Bit-reproducible and independent of how the points are batched."""
        _, dens, proj = self._query_radiance_dirs(means, covs, dirs, table, raw, colors=False)
        return proj, dens

    def _query_radiance_dirs(self, means, covs, dirs, table, raw: bool, colors: bool):
        name = "query_radiance_dirs" if colors else "query_radiance_proj"
        shape, m, c, _, dd, tab = _query_points(name, means, covs, None, dirs, table)
        if not self.use_viewdirs:
            raise NotImplementedError(f"{name}: the model has use_viewdirs=False (its colour does not depend on the "
                                      "direction; use query_radiance)")
        if self._builds_graph():
            raise NotImplementedError(f"{name}: no gradients; call it under torch.no_grad() on an autograd model")
        with torch.no_grad():
            dev = _dev(m)
            p, nd = m.shape[0], dd.shape[0]
            k = tab.shape[1] if tab is not None else 0
            prec = _cabi.PRECISIONS[self.precision]
            cfg = self._config()
            ws, keep = self.mlp._weights_struct(cfg, prec, dev)
            out_rgb = torch.empty(p, nd, 3, device=dev) if colors else None
            out_dens = torch.empty(p, device=dev)
            proj = torch.empty(p, k, 3, device=dev) if tab is not None else None
            if p > 0:
                lib = _cabi.lib()
                nbytes = lib.mipnerf_b200_radiance_dirs_workspace_bytes(C.byref(cfg), p, nd, prec)
                if nbytes == 0:
                    raise NotImplementedError(f"{name}: precision {self.precision!r} does not take this model")
                scratch = _Workspace.get(dev, nbytes)
                rgb_ptr = _ptr(out_rgb)
                _call(dev, f"MipNerf.{name}", lib.mipnerf_b200_query_radiance_dirs, C.byref(cfg), C.byref(ws),
                      m.data_ptr(), _ptr(c), p, dd.data_ptr(), nd, prec, rgb_ptr if raw else None,
                      None if raw else rgb_ptr, out_dens.data_ptr() if raw else None,
                      None if raw else out_dens.data_ptr(), _ptr(tab), k, int(raw), _ptr(proj), scratch.data_ptr(),
                      scratch.numel())
        return (out_rgb.reshape(*shape, nd, 3) if colors else None, out_dens.reshape(shape),
                proj.reshape(*shape, k, 3) if proj is not None else None)

    def _forward(self, rays: Rays, randomized: bool, white_bkgd: bool, t_rand, u_jitter, density_normal,
                 return_inds: bool):
        """The launches of `forward` -> (LevelOutputs, config, rng or None, per-level density normals or None,
        the fp32 ray tensors handed to the library)."""
        if self.ray_shape == 'cylinder':
            raise NotImplementedError  # models/mip.py:97-98
        assert self.ray_shape == 'cone'
        if self.use_viewdirs and not self._append_identity:
            raise RuntimeError("append_identity=False: view encoding width does not match view_layers "
                               "(same failure as the reference)")
        dev = _dev(rays.origins)
        b = rays.origins.shape[0]
        prec = _cabi.PRECISIONS[self.precision]
        cfg = self._config()
        rs, keep = _rays_struct(rays.origins, rays.directions, rays.viewdirs, rays.radii, rays.near, rays.far)
        rng, t_rand, u_jitter, normals = self._noise(randomized, b, dev, t_rand, u_jitter, density_normal)
        ws, wkeep = self.mlp._weights_struct(cfg, prec, dev)
        ret, outs = _level_outputs(b, self.num_samples, self.num_levels, dev, normals, return_inds)
        lib = _cabi.lib()
        # a config the library refuses sizes no workspace; the call below then raises the refusal
        scratch = _Workspace.get(dev, lib.mipnerf_b200_workspace_bytes(C.byref(cfg), b, prec))
        if rng is not None:
            _call(dev, "MipNerf.forward", lib.mipnerf_b200_forward_rng, C.byref(cfg), C.byref(ws), C.byref(rs),
                  C.byref(rng), int(bool(white_bkgd)), prec, outs, scratch.data_ptr(), scratch.numel())
        else:
            _call(dev, "MipNerf.forward", lib.mipnerf_b200_forward, C.byref(cfg), C.byref(ws), C.byref(rs),
                  int(bool(randomized)), _ptr(t_rand), _ptr(u_jitter), int(bool(white_bkgd)), prec, outs,
                  scratch.data_ptr(), scratch.numel())
        return ret, cfg, rng, normals, keep


def _check_autograd_precision(model: MipNerf, what: str) -> None:
    """The precisions a backward pass from arbitrary cotangents takes: fp32 and bf16."""
    if model.precision in ("fp16x3", "bf16x3"):
        raise NotImplementedError(f"{what}: precision={model.precision!r} is forward-only; use 'fp32' or 'bf16'")
    if model.precision == "fp16":
        raise NotImplementedError(f"{what}: fp16's fixed gradient scale is sized for the reference loss and arbitrary "
                                  "losses can overflow or underflow it; use precision='bf16'")
    if model.precision not in ("fp32", "bf16"):
        raise ValueError(f"precision={model.precision!r}")


def _check_autograd(model: MipNerf, rays: Rays, b: int) -> None:
    """Refuse, at forward time, what the backward pass cannot differentiate."""
    _check_autograd_precision(model, "MipNerf(autograd=True)")
    if not model.stop_resample_grad:
        raise NotImplementedError("MipNerf(autograd=True): gradients through the resampled fenceposts "
                                  "(stop_resample_grad=False) are not implemented")
    if any(isinstance(x, torch.Tensor) and x.requires_grad for x in rays):
        raise NotImplementedError("MipNerf(autograd=True): gradients with respect to the rays are not implemented; "
                                  "pass ray tensors that do not require grad")
    cfg = model._config()
    lib = _cabi.lib()
    if lib.mipnerf_b200_train_workspace_bytes(C.byref(cfg), max(b, 1)) == 0:
        raise NotImplementedError(f"MipNerf(autograd=True): {_cabi.last_error() or 'no training kernels'}; the "
                                  "backward pass needs use_viewdirs=True with one view layer and net_depth <= 16")
    if model.precision == "bf16" and lib.mipnerf_b200_train_workspace_bytes_for(C.byref(cfg), max(b, 1), _cabi.BF16) == 0:
        raise NotImplementedError("MipNerf(autograd=True, precision='bf16'): the tensor-core backward supports the "
                                  "8x256 / 1x128 MLP with max_deg_point=16, deg_view=4; use precision='fp32'")


def _forward_with_grad(model: MipNerf, rays: Rays, randomized, white_bkgd, t_rand, u_jitter, density_normal,
                       return_inds):
    _dev(rays.origins)
    _check_autograd(model, rays, rays.origins.shape[0])
    holder = {}
    flat = _ForwardWithGrad.apply(model, rays, randomized, white_bkgd, t_rand, u_jitter, density_normal,
                                  return_inds, holder, *model.mlp.params())
    per = 6 if return_inds else 5
    ret = LevelOutputs(tuple(flat[i:i + per]) for i in range(0, len(flat), per))
    ret.pixels = holder["pixels"]
    return ret


class _ForwardWithGrad(torch.autograd.Function):
    """MipNerf.forward as a function of the 24 MLP tensors.  Saved: the rays, each level's fenceposts, the density
    noise (Philox seed / offset or the normals) and the parameters; backward re-evaluates the MLP at those fenceposts
    and runs the library's backward chain from the output cotangents."""

    @staticmethod
    def forward(ctx, model, rays, randomized, white_bkgd, t_rand, u_jitter, density_normal, return_inds, holder,
                *params):
        ret, cfg, rng, normals, keep = model._forward(rays, randomized, white_bkgd, t_rand, u_jitter, density_normal,
                                                      return_inds)
        holder["pixels"] = ret.pixels
        levels = len(ret)
        ts = [lvl[4] for lvl in ret]
        given = [x for x in normals if x is not None]
        ctx.model, ctx.cfg, ctx.white_bkgd = model, cfg, bool(white_bkgd)
        ctx.randomized, ctx.precision, ctx.levels, ctx.per = bool(randomized), model.precision, levels, len(ret[0])
        ctx.rng = None if rng is None else (rng.seed, rng.offset)
        ctx.normal_levels = [i for i, x in enumerate(normals) if x is not None]
        ctx.num_params = len(params)
        ctx.save_for_backward(*params, *keep, *ts, *given)
        ctx.set_materialize_grads(False)
        outs = [x for lvl in ret for x in lvl]
        ctx.mark_non_differentiable(*[x for lvl in ret for x in lvl[4:] if x is not None])
        return tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        saved = ctx.saved_tensors  # raises if a parameter was updated in place since the forward
        np_, levels, per = ctx.num_params, ctx.levels, ctx.per
        params = saved[:np_]
        keep = saved[np_:np_ + 6]
        ts = saved[np_ + 6:np_ + 6 + levels]
        given = saved[np_ + 6 + levels:]
        model, cfg = ctx.model, ctx.cfg
        dev = keep[0].device
        b = keep[0].shape[0]
        out_grads = [torch.empty_like(p) for p in params]
        if all(g is None for g in grads) or b == 0:
            return (None,) * 9 + tuple(g.zero_() for g in out_grads)
        rs, _ = _rays_struct(*keep)
        cots = (_cabi.LevelCotangent * levels)()
        cot_keep = []
        for lvl in range(levels):
            ptrs = []
            for g in grads[lvl * per:lvl * per + 4]:
                if g is None:
                    ptrs.append(None)
                else:
                    g = _f32(g)
                    cot_keep.append(g)
                    ptrs.append(g.data_ptr())
            cots[lvl] = _cabi.LevelCotangent(*ptrs)
        t_arr = (C.c_void_p * levels)(*[t.data_ptr() for t in ts])
        normal_arr = None
        if ctx.normal_levels:
            normal_arr = (C.c_void_p * levels)()
            for i, x in zip(ctx.normal_levels, given):
                normal_arr[i] = x.data_ptr()
        rng = _cabi.Rng(*ctx.rng) if ctx.rng is not None else None
        ws, wkeep = model.mlp._weights_struct(cfg, _cabi.FP32, dev)
        garr = _grad_array(out_grads)
        lib = _cabi.lib()
        nbytes = lib.mipnerf_b200_train_workspace_bytes(C.byref(cfg), b)
        scratch = _Workspace.get(dev, nbytes)
        _call(dev, "MipNerf.backward", lib.mipnerf_b200_backward, C.byref(cfg), C.byref(ws), C.byref(rs), t_arr,
              int(ctx.randomized), C.byref(rng) if rng is not None else None, normal_arr, int(ctx.white_bkgd),
              _cabi.PRECISIONS[ctx.precision], cots, garr, len(garr), 0, scratch.data_ptr(), scratch.numel())
        return (None,) * 9 + tuple(out_grads)


def _check_query_autograd(model: MipNerf, tensors, radiance: bool) -> None:
    """Refuse, at query time, what the query backward cannot differentiate."""
    _check_autograd_precision(model, "MipNerf(autograd=True) queries")
    if any(isinstance(x, torch.Tensor) and x.requires_grad for x in tensors):
        raise NotImplementedError("MipNerf(autograd=True) queries: gradients with respect to means, covs or viewdirs "
                                  "are not implemented; pass tensors that do not require grad")
    cfg = model._config()
    lib = _cabi.lib()
    if lib.mipnerf_b200_query_backward_workspace_bytes(C.byref(cfg), 1, int(radiance),
                                                       _cabi.PRECISIONS[model.precision]) == 0:
        raise NotImplementedError("MipNerf(autograd=True) queries: the backward needs use_viewdirs=True with one view "
                                  "layer and net_depth <= 16, and in bf16 the 8x256 / 1x128 MLP with max_deg_point=16, "
                                  "deg_view=4; use precision='fp32' or autograd=False")


def _query_with_grad(model: MipNerf, given, shape, m, c, v, raw: bool):
    """A query with a grad_fn, on the output of `_query_points`; `given` are the caller's tensors."""
    radiance = v is not None
    _check_query_autograd(model, given, radiance)
    outs = _QueryWithGrad.apply(model, m, c, v, bool(raw), *model.mlp.params())
    if not radiance:
        return outs[0].reshape(shape)
    return outs[0].reshape(*shape, 3), outs[1].reshape(shape)


class _QueryWithGrad(torch.autograd.Function):
    """query_density (viewdirs None) / query_radiance as a function of the 24 MLP tensors.  Saved: the flattened fp32
    means, covs and viewdirs and the parameters; backward re-evaluates the field at those points with every activation
    kept and runs the library's backward chain from the output cotangents (mipnerf_b200_query_backward)."""

    @staticmethod
    def forward(ctx, model, means, covs, viewdirs, raw, *params):
        radiance = viewdirs is not None
        if radiance:
            outs = model._query_radiance(means, covs, viewdirs, raw)
        else:
            outs = (model._query_density(means, covs, raw),)
        ctx.model, ctx.cfg, ctx.raw, ctx.radiance = model, model._config(), raw, radiance
        ctx.precision = model.precision
        ctx.save_for_backward(means, covs, viewdirs, *params)
        ctx.set_materialize_grads(False)
        return outs

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        saved = ctx.saved_tensors  # raises if a parameter was updated in place since the forward
        means, covs, viewdirs = saved[:3]
        params = saved[3:]
        dev = means.device
        p = means.shape[0]
        out_grads = [torch.empty_like(x) for x in params]
        if all(g is None for g in grads) or p == 0:
            return (None,) * 5 + tuple(g.zero_() for g in out_grads)
        keep = [None if g is None else _f32(g).reshape(-1) for g in grads]
        if ctx.radiance:
            pair = (_ptr(keep[0]), _ptr(keep[1]))
            cot = _cabi.QueryCotangent(*pair, None, None) if ctx.raw else _cabi.QueryCotangent(None, None, *pair)
        else:
            cot = _cabi.QueryCotangent(None, _ptr(keep[0]), None, None) if ctx.raw else \
                _cabi.QueryCotangent(None, None, None, _ptr(keep[0]))
        model, cfg = ctx.model, ctx.cfg
        prec = _cabi.PRECISIONS[ctx.precision]
        ws, wkeep = model.mlp._weights_struct(cfg, _cabi.FP32, dev)
        garr = _grad_array(out_grads)
        lib = _cabi.lib()
        nbytes = lib.mipnerf_b200_query_backward_workspace_bytes(C.byref(cfg), p, int(ctx.radiance), prec)
        # per call, not the per-stream _Workspace: up to one chunk's activations (GBs), which a forward-only process
        # that ran one query backward should not keep reserved for small forwards
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        _call(dev, "MipNerf.query backward", lib.mipnerf_b200_query_backward, C.byref(cfg), C.byref(ws),
              means.data_ptr(), _ptr(covs), _ptr(viewdirs), p, prec, C.byref(cot), garr, len(garr), 0,
              scratch.data_ptr(), scratch.numel())
        return (None,) * 5 + tuple(out_grads)
