"""float64 torch restatement of the baked-grid renderer (tests/grid_render_ref.py), differentiable in each level's
parameters: the kept points' densities [M_l] in SH-row order and their SH rows [M_l, (degree + 1)^2, 3].

The fp32 sample lattice, the inside test and the level choice are grid_render_ref's, computed in numpy; the
interpolation, the SH sum, the sigmoid and the compositing are float64 torch.  As the kernel's backward does, samples
in empty macro cells (found by the kernel's fp32 cell lookup, only for dt > 0) and samples after the one that stops
the ray are detached.  Also returned per ray: the smallest |T_after / 1e-4 - 1| over the samples up to the stop, so
that a test can leave out rays whose stop is within rounding of the threshold."""
import numpy as np
import torch

import grid_render_ref as ref
from mipnerf_pl_b200.field import sh_basis

f32 = np.float32


def lattice(kept, index, fill_shape=()):
    """[nz, ny, nx, *fill_shape] float64: `kept` [M, *fill_shape] at the points whose index is r, 0 where -1."""
    idx = torch.as_tensor(np.asarray(index), dtype=torch.int64)
    out = torch.zeros(idx.shape + tuple(fill_shape), dtype=torch.float64)
    keep = idx >= 0
    return out.index_put((keep.nonzero(as_tuple=True)), kept[idx[keep]])


def trilinear(values, lo, hi, x):
    """ref.trilinear in torch: values [nz, ny, nx, ...], x [..., 3] float64 numpy -> [..., ...]."""
    n = np.array(values.shape[:3][::-1])
    u = np.clip((x - lo) / (hi - lo) * (n - 1), 0, n - 1)
    i = np.minimum(np.floor(u).astype(np.int64), n - 2)
    f = u - i
    out = 0.0
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
        w = (f[..., 0] if dx else 1 - f[..., 0]) * (f[..., 1] if dy else 1 - f[..., 1]) * \
            (f[..., 2] if dz else 1 - f[..., 2])
        v = values[torch.as_tensor(i[..., 2] + dz), torch.as_tensor(i[..., 1] + dy), torch.as_tensor(i[..., 0] + dx)]
        w = torch.as_tensor(w)
        out = out + w.reshape(w.shape + (1,) * (v.dim() - w.dim())) * v
    return out


def empty_cells(occupancy, block, n0, bounds, x32):
    """[...] bool: the kernel's fp32 macro-cell lookup of positions x32 [..., 3] finds an empty cell."""
    lo, hi = np.asarray(bounds[0], f32), np.asarray(bounds[1], f32)
    occ = np.asarray(occupancy)
    c = []
    for a in range(3):
        inv_s = f32(n0[a] - 1) / (hi[a] - lo[a])
        u = np.minimum(np.maximum((x32[..., a] - lo[a]) * inv_s, f32(0)), f32(n0[a] - 2))
        c.append(u.astype(np.int64) // block)
    return occ[c[2], c[1], c[0]] == 0


def render(params, indices, occupancy, block, bounds, degree, rgb_padding, origins, directions, viewdirs, radii, near,
           far, step, white_bkgd, chunk=256):
    """params: [(kept density [M_l], sh [M_l, K, 3])] float64 torch; indices: per level [nz, ny, nx] (row or -1);
    occupancy [oz, oy, ox] -> (rgb [B,3], distance [B], acc [B], stop margin [B] numpy)."""
    lo64, hi64 = np.asarray(bounds[0], np.float64), np.asarray(bounds[1], np.float64)
    lo32, hi32 = np.asarray(bounds[0], f32), np.asarray(bounds[1], f32)
    L = len(params)
    nc = (degree + 1) ** 2
    dens = [lattice(kd, idx) for (kd, _), idx in zip(params, indices)]
    coef = [lattice(sh, idx, (nc, 3)) for (_, sh), idx in zip(params, indices)]
    n0 = np.array(np.asarray(indices[0]).shape[::-1])
    s0 = float(np.max((hi64 - lo64) / (n0 - 1)))
    p = float(f32(rgb_padding))
    o32, d32 = np.asarray(origins, f32).reshape(-1, 3), np.asarray(directions, f32).reshape(-1, 3)
    near32, far32 = np.asarray(near, f32).reshape(-1), np.asarray(far, f32).reshape(-1)
    B = o32.shape[0]
    K, dt, dn = ref.sample_lattice(d32, near32, far32, step)
    Y = torch.as_tensor(sh_basis(np.asarray(viewdirs, np.float64).reshape(-1, 3), degree))  # [B, nc]
    rad = np.asarray(radii, np.float64).reshape(-1)
    rgbs, dists, accs, margins = [], [], [], []
    for c0 in range(0, B, chunk):
        sl = slice(c0, min(B, c0 + chunk))
        kmax = int(K[sl].max())
        k = np.arange(kmax)
        valid = k[None, :] < K[sl, None]
        t32 = near32[sl, None] + (k.astype(f32)[None, :] + f32(0.5)) * dt[sl, None]
        x32 = o32[sl, None, :] + t32[..., None] * d32[sl, None, :]
        inside = valid & np.all((x32 >= lo32) & (x32 <= hi32), axis=-1)
        skipped = inside & (dt[sl, None] > 0) & empty_cells(occupancy, block, n0, bounds, x32)
        t = t32.astype(np.float64)
        x = o32[sl, None, :].astype(np.float64) + t[..., None] * d32[sl, None, :].astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.log2(np.sqrt(3.0) * rad[sl, None] * t / s0)
        lam = np.clip(np.nan_to_num(lam, nan=0.0, neginf=0.0, posinf=L - 1), 0, L - 1)
        a = np.minimum(np.floor(lam).astype(np.int64), L - 1)
        f = np.where(a == L - 1, 0.0, lam - a)
        sigma = torch.zeros(t.shape, dtype=torch.float64)
        raw = torch.zeros(t.shape + (3,), dtype=torch.float64)
        for lvl in range(L):
            wl = np.where(a == lvl, 1 - f, 0.0) + np.where(a + 1 == lvl, f, 0.0)
            if not np.any(wl[inside] > 0):
                continue
            wl = torch.as_tensor(wl)
            sigma = sigma + wl * trilinear(dens[lvl], lo64, hi64, x)
            cl = trilinear(coef[lvl], lo64, hi64, x)  # [R, k, nc, 3]
            raw = raw + wl[..., None] * torch.einsum("rkjc,rj->rkc", cl, Y[sl])
        ins, skp = torch.as_tensor(inside), torch.as_tensor(skipped)
        sigma = torch.where(ins, sigma, torch.zeros((), dtype=torch.float64))
        sigma = torch.where(skp, sigma.detach(), sigma)
        col = (1 + 2 * p) * torch.sigmoid(raw) - p
        delta = torch.as_tensor((dt[sl].astype(np.float64) * dn[sl].astype(np.float64))[:, None])
        alpha = 1 - torch.exp(-sigma * delta)
        T_after = torch.cumprod(1 - alpha, dim=1)
        T_before = torch.cat([torch.ones(T_after.shape[0], 1, dtype=torch.float64), T_after[:, :-1]], dim=1)
        below = (T_after < ref.STOP_T).numpy()
        stopped = np.concatenate([np.zeros((below.shape[0], 1), bool), np.cumsum(below, axis=1)[:, :-1] > 0], axis=1)
        live = inside & ~stopped
        w = torch.where(torch.as_tensor(live), T_before * alpha, torch.zeros((), dtype=torch.float64))
        rgbs.append(torch.einsum("rk,rkc->rc", w, col))
        accs.append(w.sum(1))
        dists.append((w * torch.as_tensor(t)).sum(1))
        gap = np.abs(T_after.detach().numpy() / ref.STOP_T - 1)
        margins.append(np.where(live, gap, np.inf).min(axis=1, initial=np.inf))
    if B == 0:
        z = torch.zeros(0, dtype=torch.float64)
        return torch.zeros(0, 3, dtype=torch.float64), z, z, np.zeros(0)
    rgb, dist, acc = torch.cat(rgbs), torch.cat(dists), torch.cat(accs)
    dist = torch.clamp(dist, torch.as_tensor(near32.astype(np.float64)), torch.as_tensor(far32.astype(np.float64)))
    if white_bkgd:
        rgb = rgb + (1 - acc)[:, None]
    return rgb, dist, acc, np.concatenate(margins)
