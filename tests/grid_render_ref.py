"""numpy float64 restatement of the baked-grid renderer (include/mipnerf_b200.h, mipnerf_b200_grid_render) and of
trilinear interpolation on a baked level.

K, dt and t_k are computed as the contract states them, in fp32 (each numpy float32 operation rounds once, as the
kernel's explicitly rounded ones do); so is the sample position o + t_k d that decides whether a sample is inside the
bounds.  Everything else (interpolation, level blend, SH, compositing, termination) is float64, and every sample is
marched: no clipping, no skipping."""
import numpy as np

from mipnerf_pl_b200.field import sh_basis

STOP_T = 1e-4
f32 = np.float32


def sample_lattice(directions, near, far, step):
    """-> (K [B] int64, dt [B] fp32, |d| [B] fp32) by the fp32 formulas."""
    d = np.asarray(directions, dtype=f32)
    dn = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    near, far = np.asarray(near, dtype=f32).reshape(-1), np.asarray(far, dtype=f32).reshape(-1)
    span = far - near
    kf = np.ceil(span * dn / f32(step))
    K = np.where(kf >= 1, kf, 1).astype(np.int64)
    dt = span / K.astype(f32)
    return K, dt, dn


def trilinear(values, lo, hi, x):
    """Trilinear interpolation of values [nz, ny, nx, ...] (lattice over [lo, hi]) at points x [..., 3] (float64),
    coordinates clamped to the lattice; -> [..., ...]."""
    n = np.array(values.shape[:3][::-1])
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    u = np.clip((x - lo) / (hi - lo) * (n - 1), 0, n - 1)
    i = np.minimum(np.floor(u).astype(np.int64), n - 2)
    f = u - i
    out = 0.0
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
        w = (f[..., 0] if dx else 1 - f[..., 0]) * (f[..., 1] if dy else 1 - f[..., 1]) * \
            (f[..., 2] if dz else 1 - f[..., 2])
        v = values[i[..., 2] + dz, i[..., 1] + dy, i[..., 0] + dx]
        out = out + w.reshape(w.shape + (1,) * (v.ndim - w.ndim)) * v
    return out


def coefficient_lattice(index, sh):
    """[nz, ny, nx, K, 3] float64: the SH rows of kept points, 0 where the index is -1."""
    k = sh.shape[1] if sh.ndim == 3 else 1
    out = np.zeros(index.shape + (k, 3))
    kept = index >= 0
    out[kept] = np.asarray(sh, np.float64)[index[kept]]
    return out


def render(levels, bounds, degree, rgb_padding, origins, directions, viewdirs, radii, near, far, step, white_bkgd,
           chunk=512):
    """levels: [(density [nz, ny, nx], index [nz, ny, nx], sh [M, K, 3])] -> (rgb [B,3], distance [B], acc [B]) float64."""
    lo64, hi64 = np.asarray(bounds[0], np.float64), np.asarray(bounds[1], np.float64)
    lo32, hi32 = np.asarray(bounds[0], f32), np.asarray(bounds[1], f32)
    L = len(levels)
    dens = [np.asarray(d, np.float64) for d, _, _ in levels]
    coef = [coefficient_lattice(np.asarray(i), np.asarray(s)) for _, i, s in levels]
    n0 = np.array(dens[0].shape[::-1])
    s0 = float(np.max((hi64 - lo64) / (n0 - 1)))
    p = float(f32(rgb_padding))
    o32, d32 = np.asarray(origins, f32).reshape(-1, 3), np.asarray(directions, f32).reshape(-1, 3)
    near32, far32 = np.asarray(near, f32).reshape(-1), np.asarray(far, f32).reshape(-1)
    B = o32.shape[0]
    K, dt, dn = sample_lattice(d32, near32, far32, step)
    Y = sh_basis(np.asarray(viewdirs, np.float64).reshape(-1, 3), degree)  # [B, Kc]
    rad = np.asarray(radii, np.float64).reshape(-1)
    rgb, dist, acc = np.zeros((B, 3)), np.zeros(B), np.zeros(B)
    for c0 in range(0, B, chunk):
        sl = slice(c0, min(B, c0 + chunk))
        kmax = int(K[sl].max()) if B else 0
        k = np.arange(kmax)
        valid = k[None, :] < K[sl, None]
        t32 = near32[sl, None] + (k.astype(f32)[None, :] + f32(0.5)) * dt[sl, None]   # fp32, rounded per op
        x32 = o32[sl, None, :] + t32[..., None] * d32[sl, None, :]
        inside = valid & np.all((x32 >= lo32) & (x32 <= hi32), axis=-1)
        t = t32.astype(np.float64)
        x = o32[sl, None, :].astype(np.float64) + t[..., None] * d32[sl, None, :].astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.log2(np.sqrt(3.0) * rad[sl, None] * t / s0)
        lam = np.clip(np.nan_to_num(lam, nan=0.0, neginf=0.0, posinf=L - 1), 0, L - 1)
        a = np.minimum(np.floor(lam).astype(np.int64), L - 1)
        f = np.where(a == L - 1, 0.0, lam - a)
        sigma = np.zeros(t.shape)
        raw = np.zeros(t.shape + (3,))
        for lvl in range(L):
            wl = np.where(a == lvl, 1 - f, 0.0) + np.where(a + 1 == lvl, f, 0.0)
            if not np.any(wl[inside] > 0):
                continue
            sigma += wl * trilinear(dens[lvl], lo64, hi64, x)
            c = trilinear(coef[lvl], lo64, hi64, x)  # [R, k, Kc, 3]
            raw += wl[..., None] * np.einsum("rkjc,rj->rkc", c, Y[sl])
        sigma = np.where(inside, sigma, 0.0)
        col = (1 + 2 * p) / (1 + np.exp(-raw)) - p
        delta = (dt[sl].astype(np.float64) * dn[sl].astype(np.float64))[:, None]
        alpha = 1 - np.exp(-sigma * delta)
        T_after = np.cumprod(1 - alpha, axis=1)
        T_before = np.concatenate([np.ones((T_after.shape[0], 1)), T_after[:, :-1]], axis=1)
        # termination: samples after the first one that leaves T < 1e-4 do not count
        stopped = np.concatenate([np.zeros((T_after.shape[0], 1), bool), np.cumsum(T_after < STOP_T, axis=1)[:, :-1] > 0],
                                 axis=1)
        w = np.where(stopped | ~inside, 0.0, T_before * alpha)
        rgb[sl] = np.einsum("rk,rkc->rc", w, col)
        acc[sl] = w.sum(1)
        dist[sl] = (w * t).sum(1)
    dist = np.minimum(np.maximum(dist, near32.astype(np.float64)), far32.astype(np.float64))
    if white_bkgd:
        rgb = rgb + (1 - acc)[:, None]
    return rgb, dist, acc
