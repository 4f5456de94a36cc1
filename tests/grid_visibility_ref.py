"""float64 restatement of mipnerf_b200_grid_visibility (include/mipnerf_b200.h): per kept point of each level, the
largest score w_k * (lw * wc_c) over the composited samples of the rays, on grid_render_ref's march.

The fp32 sample lattice and inside test are grid_render_ref's.  The level choice lambda = log2(sqrt(3) radii t_k / s_0)
and the lattice coordinates of the sample positions are the kernel's fp32 formulas: the fractional part of each is a
weight (of the upper level, of a corner), and where it is small its fp32 rounding, which the renderer applies to the
colour as well, is a large part of it.  The weights' products, the densities and the compositing are float64, and
every sample is marched (no clipping, no skipping: a skipped sample has density 0 at every level, so it scores
nothing).  Also returned per
ray: the smallest |T_after / 1e-4 - 1| over the samples up to the stop, so that a test can leave out rays whose stop
is within rounding of the threshold."""
import numpy as np

import grid_render_ref as ref

f32 = np.float32


def corners(n, lo, hi, x):
    """The 8 trilinear corners of fp32 positions x [..., 3] on a lattice of n = (nx, ny, nz) points over the fp32
    bounds [lo, hi], from the kernel's fp32 lattice coordinates u = clamp((x - lo) (n - 1) / (hi - lo), 0, n - 1):
    -> [(flat index [...] int64, weight [...] float64)] x 8."""
    n = np.asarray(n)
    inv_s = (n - 1).astype(f32) / (hi - lo)
    u = np.minimum(np.maximum((x - lo) * inv_s, f32(0)), (n - 1).astype(f32))
    i = np.minimum(u.astype(np.int64), n - 2)
    f = (u - i.astype(f32)).astype(np.float64)
    out = []
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
        w = (f[..., 0] if dx else 1 - f[..., 0]) * (f[..., 1] if dy else 1 - f[..., 1]) * \
            (f[..., 2] if dz else 1 - f[..., 2])
        out.append((((i[..., 2] + dz) * n[1] + i[..., 1] + dy) * n[0] + i[..., 0] + dx, w))
    return out


def visibility(levels, bounds, origins, directions, radii, near, far, step, chunk=512):
    """levels: [(density [nz, ny, nx], index [nz, ny, nx])] -> (per level the max scores [M_l] float64, indexed by
    SH row; per level the largest lw * wc_c and the largest w_k * wc_c over its kept corners, the scores without the
    blending weight and without the level weight; stop margin [B])."""
    lo32, hi32 = np.asarray(bounds[0], f32), np.asarray(bounds[1], f32)
    L = len(levels)
    dens = [np.asarray(d, np.float64) for d, _ in levels]
    index = [np.asarray(i).reshape(-1) for _, i in levels]
    shapes = [d.shape[::-1] for d in dens]  # (nx, ny, nz)
    out = [np.zeros(int((i >= 0).sum())) for i in index]
    coef, unweighted = [0.0] * L, [0.0] * L
    s0 = np.max((hi32 - lo32) / (np.array(shapes[0]) - 1).astype(f32))  # fp32, as the kernel's s0_max
    o32, d32 = np.asarray(origins, f32).reshape(-1, 3), np.asarray(directions, f32).reshape(-1, 3)
    near32, far32 = np.asarray(near, f32).reshape(-1), np.asarray(far, f32).reshape(-1)
    B = o32.shape[0]
    K, dt, dn = ref.sample_lattice(d32, near32, far32, step)
    rad = np.asarray(radii, f32).reshape(-1)
    margins = []
    for c0 in range(0, B, chunk):
        sl = slice(c0, min(B, c0 + chunk))
        k = np.arange(int(K[sl].max()))
        valid = k[None, :] < K[sl, None]
        t32 = near32[sl, None] + (k.astype(f32)[None, :] + f32(0.5)) * dt[sl, None]
        x32 = o32[sl, None, :] + t32[..., None] * d32[sl, None, :]
        inside = valid & np.all((x32 >= lo32) & (x32 <= hi32), axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.log2(f32(np.sqrt(3.0)) * rad[sl, None] * t32 / s0)
        lam = np.clip(np.nan_to_num(lam, nan=0.0, neginf=0.0, posinf=L - 1), f32(0), f32(L - 1))
        a = np.minimum(np.floor(lam).astype(np.int64), L - 1)
        f = np.where(a == L - 1, 0.0, (lam - a.astype(f32)).astype(np.float64))
        wl = [np.where(a == lvl, 1 - f, 0.0) + np.where(a + 1 == lvl, f, 0.0) for lvl in range(L)]
        sigma = np.zeros(t32.shape)
        cs = [None] * L
        for lvl in range(L):
            if not np.any(wl[lvl][inside] > 0):
                continue
            cs[lvl] = corners(shapes[lvl], lo32, hi32, x32)
            flat = dens[lvl].reshape(-1)
            sigma += wl[lvl] * sum(w * flat[p] for p, w in cs[lvl])
        sigma = np.where(inside, sigma, 0.0)
        delta = (dt[sl].astype(np.float64) * dn[sl].astype(np.float64))[:, None]
        alpha = 1 - np.exp(-sigma * delta)
        T_after = np.cumprod(1 - alpha, axis=1)
        T_before = np.concatenate([np.ones((T_after.shape[0], 1)), T_after[:, :-1]], axis=1)
        below = T_after < ref.STOP_T
        stopped = np.concatenate([np.zeros((below.shape[0], 1), bool), np.cumsum(below, axis=1)[:, :-1] > 0], axis=1)
        live = inside & ~stopped
        w = np.where(live, T_before * alpha, 0.0)
        for lvl in range(L):
            if cs[lvl] is None:
                continue
            for p, wc in cs[lvl]:
                row = index[lvl][p]
                sel = live & (row >= 0) & (wl[lvl] > 0)
                np.maximum.at(out[lvl], row[sel], (w * wl[lvl] * wc)[sel])
                coef[lvl] = max(coef[lvl], float((wl[lvl] * wc)[sel].max(initial=0.0)))
                unweighted[lvl] = max(unweighted[lvl], float((w * wc)[sel].max(initial=0.0)))
        gap = np.abs(T_after / ref.STOP_T - 1)
        margins.append(np.where(live, gap, np.inf).min(axis=1, initial=np.inf))
    return out, (coef, unweighted), (np.concatenate(margins) if margins else np.zeros(0))
