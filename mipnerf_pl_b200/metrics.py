"""Image metrics and the evaluation / video render loops of the reference on the device.

* `eval_errors(pred, target)` -> (psnr, ssim): utils/metrics.py:190-197 (PSNR :182-188; Gaussian-window SSIM :44-126)
  as ONE library call per frame (`mipnerf_b200_image_metrics`), no five full-size conv2d maps.
* `evaluate(system, dataset)`: eval.py:49-84 — every test image through `render_image`, PSNR / SSIM per image,
  `psnrs.txt` / `ssims.txt`, optional PNGs (utils/vis.py:66-89).  The reference unpacks 3 of the forward's 5 tuple
  fields there (eval.py:61) and fails; this loop reads the tuple correctly.
* `render_path(model, ...)`: render_video.py:115-153 — the 120-pose spheric path (utils/vis.py:159-198) with rays
  generated on the device and frame rows sharded over the ranks; returns the per-frame device time.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _cabi
from .ops import _call, _dev, _f32
from .rays import spheric_pose


def eval_errors(pred_color: torch.Tensor, batch_pixels: torch.Tensor):
    """(psnr, ssim) of [1,H,W,3] (or [H,W,3]) CUDA images, as 0-d tensors."""
    dev = _dev(pred_color)
    p, t = _f32(pred_color), _f32(batch_pixels)
    if p.shape != t.shape:
        raise ValueError(f"img1 and img2 shapes must be the same. Got: {tuple(p.shape)} {tuple(t.shape)}")
    if p.dim() == 4:
        if p.shape[0] != 1:
            raise NotImplementedError("one frame per call (the reference's loaders use batch_size=1)")
        p, t = p[0], t[0]
    h, w, c = p.shape
    lib = _cabi.lib()
    nbytes = lib.mipnerf_b200_image_metrics_scratch_bytes(h, w, c)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out = torch.empty(3, device=dev)
    _call(dev, "eval_errors", lib.mipnerf_b200_image_metrics, p.data_ptr(), t.data_ptr(), h, w, c, scratch.data_ptr(),
          nbytes, out.data_ptr())
    return out[0], out[1]


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, reduction: str = "mean", max_val: float = 1.0):
    """utils/metrics.py:165-179 for the configuration the reference uses (window 11, mean, max_val 1); inputs BxCxHxW."""
    if window_size != 11 or reduction != "mean" or max_val != 1.0:
        raise NotImplementedError("the device kernel implements eval_errors' configuration: window 11, mean, max_val 1")
    return eval_errors(img1.permute(0, 2, 3, 1), img2.permute(0, 2, 3, 1))[1]


def visualize_depth(depth: torch.Tensor) -> np.ndarray:
    """utils/vis.py:75-89: min-max normalise, JET colour map -> uint8 [H,W,3] (RGB)."""
    import cv2
    x = np.nan_to_num(depth.detach().float().cpu().numpy().squeeze())
    mi, ma = float(x.min()), float(x.max())
    x = (255 * (x - mi) / max(ma - mi, 1e-8)).astype(np.uint8)
    return cv2.cvtColor(cv2.applyColorMap(x, cv2.COLORMAP_JET), cv2.COLOR_BGR2RGB)


def save_images(rgb: torch.Tensor, dist: torch.Tensor, acc: torch.Tensor, path: str, idx: int) -> None:
    """utils/vis.py:66-72: <idx>_rgb.png, _dist.png, _acc.png."""
    from PIL import Image
    os.makedirs(path, exist_ok=True)
    img = (rgb.detach().float().clamp(0, 1).reshape(rgb.shape[-3], rgb.shape[-2], 3).cpu().numpy() * 255).astype(np.uint8)
    Image.fromarray(img).save(os.path.join(path, f"{idx:05d}_rgb.png"))
    Image.fromarray(visualize_depth(dist)).save(os.path.join(path, f"{idx:05d}_dist.png"))
    Image.fromarray(visualize_depth(acc)).save(os.path.join(path, f"{idx:05d}_acc.png"))


@torch.no_grad()
def evaluate(system, dataset, out_dir: Optional[str] = None, save_image: bool = False, max_images: Optional[int] = None):
    """eval.py:49-84 over a `single_image` dataset of (Rays [H,W,.], rgbs [H,W,3]) items."""
    dev = next(system.parameters()).device
    psnrs: List[float] = []
    ssims: List[float] = []
    n = len(dataset) if max_images is None else min(len(dataset), max_images)
    for idx in range(n):
        rays, rgbs = dataset[idx]
        rays = type(rays)(*[torch.as_tensor(f)[None].to(dev) for f in rays])
        rgbs = torch.as_tensor(rgbs)[None].to(dev)
        _, fine, _, dist = system.render_image((rays, rgbs), return_distance=True)
        psnr, ss = eval_errors(fine, rgbs[..., :3])
        psnrs.append(float(psnr))
        ssims.append(float(ss))
        if out_dir and save_image:
            save_images(fine, dist, dist, os.path.join(out_dir, "images"), idx)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "psnrs.txt"), "w") as f:
            f.write(" ".join(str(v) for v in psnrs))
        with open(os.path.join(out_dir, "ssims.txt"), "w") as f:
            f.write(" ".join(str(v) for v in ssims))
    return psnrs, ssims


def spheric_path(n_poses: int = 120, radius: float = 4.0, phi: float = -np.pi / 5) -> np.ndarray:
    """utils/vis.py:159-198 `create_spheric_poses`: n_poses camera-to-world [3,4] on the circle."""
    return np.stack([spheric_pose(float(th), phi, radius) for th in np.linspace(0, 2 * np.pi, n_poses + 1)[:-1]], 0)


@torch.no_grad()
def render_path(model, poses: Optional[Sequence[np.ndarray]] = None, height: int = 800, width: int = 800,
                white_bkgd: bool = True, world: int = 1, rank: int = 0, group=None, out_dir: Optional[str] = None,
                n_poses: int = 120):
    """render_video.py:115-153: every pose -> (fine rgb, distance) frame; returns {'ms_per_frame': [...], 'frames': n}.
    Rays are generated on the device for this rank's rows, the rendered rows are all-gathered (render.render_frame)."""
    from .render import render_frame
    dev = next(model.parameters()).device
    poses = spheric_path(n_poses) if poses is None else poses
    times = []
    for idx, c2w in enumerate(poses):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, fine, dist = render_frame(model, c2w, height, width, white_bkgd, world=world, rank=rank, group=group, device=dev)
        e1.record()
        if out_dir and rank == 0:
            save_images(fine, dist, dist, out_dir, idx)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return {"ms_per_frame": times, "frames": len(times)}
