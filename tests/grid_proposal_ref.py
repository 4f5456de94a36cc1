"""float64 restatement of mipnerf_b200_grid_proposal (include/mipnerf_b200.h): per ray and interval of the caller's
fenceposts, the baked grid's density at the interval's midpoint, composited as volumetric_rendering's weights with no
stop.

The roundings the header fixes are reproduced in fp32: the midpoint t_mid, the position o + t_mid d, |d| and delta.
The level choice lambda = log2(sqrt(3) radii t_mid / s_0) and the lattice coordinates are the kernel's fp32 formulas,
as in grid_visibility_ref: the fractional part of each is a weight, so its fp32 rounding is part of the result.  The
densities, their products with delta, the prefix sums and the exponentials are float64.  Also returned per ray: the
sum over intervals of |sigma_a - sigma_b| delta over the two blended levels, which bounds how far a one-ulp change of
lambda's fractional part can move the optical depths."""
import numpy as np

from grid_visibility_ref import corners

f32 = np.float32


def proposal(levels, bounds, origins, directions, radii, t_samples, chunk=512):
    """levels: [density [nz, ny, nx]] (0 at dropped points) -> (weights [B, N] float64, lambda sensitivity [B])."""
    lo32, hi32 = np.asarray(bounds[0], f32), np.asarray(bounds[1], f32)
    L = len(levels)
    dens = [np.asarray(d, np.float64).reshape(-1) for d in levels]
    shapes = [np.asarray(d).shape[::-1] for d in levels]  # (nx, ny, nz)
    s0 = np.max((hi32 - lo32) / (np.array(shapes[0]) - 1).astype(f32))  # fp32, as the kernel's s0_max
    o32, d32 = np.asarray(origins, f32).reshape(-1, 3), np.asarray(directions, f32).reshape(-1, 3)
    rad = np.asarray(radii, f32).reshape(-1)
    t = np.asarray(t_samples, f32)
    B, N = t.shape[0], t.shape[1] - 1
    dn = np.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2])
    weights, sens = np.zeros((B, N)), np.zeros(B)
    for c0 in range(0, B, chunk):
        sl = slice(c0, min(B, c0 + chunk))
        with np.errstate(over="ignore", invalid="ignore"):
            tm = (t[sl, :-1] + t[sl, 1:]) * f32(0.5)
            delta = ((t[sl, 1:] - t[sl, :-1]) * dn[sl, None]).astype(np.float64)
            x32 = o32[sl, None, :] + tm[..., None] * d32[sl, None, :]
        inside = np.all((x32 >= lo32) & (x32 <= hi32), axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.log2(f32(np.sqrt(3.0)) * rad[sl, None] * tm / s0)
        lam = np.clip(np.nan_to_num(lam, nan=0.0, neginf=0.0, posinf=L - 1), f32(0), f32(L - 1))
        a = np.minimum(np.floor(lam).astype(np.int64), L - 1)
        f = np.where(a == L - 1, 0.0, (lam - a.astype(f32)).astype(np.float64))
        x32 = np.where(inside[..., None], x32, lo32)  # outside: any in-range lattice position, weighted 0 below
        per_level = [sum(w * dens[lvl][p] for p, w in corners(shapes[lvl], lo32, hi32, x32)) for lvl in range(L)]
        sig_a = np.choose(a, per_level)
        sig_b = np.choose(np.minimum(a + 1, L - 1), per_level)
        sigma = np.where(inside, (1 - f) * sig_a + f * sig_b, 0.0)
        s = sigma * delta
        depth = np.concatenate([np.zeros((s.shape[0], 1)), np.cumsum(s, axis=1)[:, :-1]], axis=1)
        weights[sl] = (1 - np.exp(-s)) * np.exp(-depth)
        sens[sl] = np.where(inside & (f > 0), np.abs(sig_a - sig_b) * delta, 0.0).sum(axis=1)
    return weights, sens
