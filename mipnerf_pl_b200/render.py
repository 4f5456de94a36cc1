"""Frame rendering on top of `MipNerf.forward`: on-device ray generation from a pose and ray-sharded
rendering across the GPUs of one node.

This is the GPU replacement for the reference's render loops (`MipNeRFSystem.render_image`
models/nerf_system.py:151-177, eval.py:49-70, render_video.py:131-152), which generate rays with
NumPy on the host, copy 33 MB per frame to the device and loop over 8192-ray chunks in Python on
one GPU.  Here a rank generates only ITS rows of the frame directly in HBM, renders them with one
C-ABI call, and the ranks exchange the rendered pixels with a single all_gather (rays are
independent, so the gathered frame is bit-identical to a single-GPU render).
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional, Sequence, Tuple

import numpy as np
import torch

from .rays import BLENDER_CAMERA_ANGLE_X, Rays


def shard_rows(height: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, near-equal row ranges: rank r renders rows [start, stop)."""
    base, extra = divmod(height, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def shard_bounds(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous, near-equal slices of a flat ray array (SURVEY.md §8e)."""
    return shard_rows(n, world, rank)


def generate_rays(c2w, height: int = 800, width: int = 800, camera_angle_x: float = BLENDER_CAMERA_ANGLE_X,
                  near: float = 2.0, far: float = 6.0, rows: Optional[Tuple[int, int]] = None,
                  device="cuda") -> Rays:
    """Rays of frame rows [rows[0], rows[1]) (default: all) as flat [R*W, C] CUDA tensors."""
    from . import _cabi
    from .ops import _call
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("generate_rays writes rays straight into HBM; use rays.blender_rays() on the host")
    r0, r1 = rows if rows is not None else (0, height)
    n = (r1 - r0) * width
    mk = lambda c: torch.empty(n, c, device=dev)  # noqa: E731
    o, d, v, rad, nr, fr = mk(3), mk(3), mk(3), mk(1), mk(1), mk(1)
    pose = np.ascontiguousarray(np.asarray(c2w, dtype=np.float32)[:3, :4]).reshape(-1)
    focal = float(np.float32(0.5 * width / np.tan(0.5 * camera_angle_x)))
    _call(dev, "generate_rays", _cabi.lib().mipnerf_b200_generate_rays, pose.ctypes.data_as(C.POINTER(C.c_float)),
          height, width, focal, near, far, r0, r1 - r0, o.data_ptr(), d.data_ptr(), v.data_ptr(), rad.data_ptr(),
          nr.data_ptr(), fr.data_ptr())
    return Rays(o, d, v, rad, torch.ones_like(rad), nr, fr)


def gather_rows(local: torch.Tensor, counts: Sequence[int], group=None) -> torch.Tensor:
    """All-gather per-rank row blocks of unequal length into the full array (one collective:
    blocks are padded to the longest and trimmed after)."""
    import torch.distributed as dist
    world = len(counts)
    if world == 1:
        return local
    longest = max(counts)
    pad = local
    if local.shape[0] < longest:
        pad = torch.cat([local, local.new_zeros((longest - local.shape[0],) + tuple(local.shape[1:]))])
    out = local.new_empty((world * longest,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, pad.contiguous(), group=group)
    return torch.cat([out[r * longest: r * longest + counts[r]] for r in range(world)])


def render_sharded(forward_fn: Callable[[Rays], Sequence[torch.Tensor]], rays: Rays, world: int, rank: int,
                   group=None):
    """Render this rank's contiguous shard of `rays` with `forward_fn` (-> per-ray tensors) and
    all-gather the results; every rank returns the full arrays."""
    n = rays.origins.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    mine = Rays(*[f[lo:hi] for f in rays])
    outs = forward_fn(mine)
    counts = [shard_bounds(n, world, r)[1] - shard_bounds(n, world, r)[0] for r in range(world)]
    return [gather_rows(o, counts, group) for o in outs]


@torch.no_grad()
def render_frame(model, c2w, height: int = 800, width: int = 800, white_bkgd: bool = True,
                 camera_angle_x: float = BLENDER_CAMERA_ANGLE_X, near: float = 2.0, far: float = 6.0,
                 world: int = 1, rank: int = 0, group=None, device=None):
    """One frame: (coarse_rgb [H,W,3], fine_rgb [H,W,3], distance [H,W]) on every rank."""
    dev = device or next(model.parameters()).device
    r0, r1 = shard_rows(height, world, rank)
    rays = generate_rays(c2w, height, width, camera_angle_x, near, far, rows=(r0, r1), device=dev)
    ret = model(rays, False, white_bkgd)
    local = torch.cat([ret[0][0], ret[-1][0], ret[-1][1][:, None]], dim=1)   # [rows*W, 7]
    counts = [(shard_rows(height, world, r)[1] - shard_rows(height, world, r)[0]) * width for r in range(world)]
    full = gather_rows(local, counts, group)
    return (full[:, 0:3].reshape(height, width, 3), full[:, 3:6].reshape(height, width, 3),
            full[:, 6].reshape(height, width))
