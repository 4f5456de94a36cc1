"""float64 restatement of mipnerf_b200_grid_proposal_backward (include/mipnerf_b200.h): the gradient of
sum_{r,i} g_ri w_ri, w = grid_proposal_ref's weights, with respect to the kept points' densities.

The fp32 roundings are grid_proposal_ref's: midpoint, position, |d|, delta, the level choice and the lattice
coordinates.  Per ray, with s_i = sigma_i delta_i and S_i = sum_{j<i} s_j, w_i = e^{-S_i} - e^{-S_{i+1}}, so
dL/ds_k = g_k e^{-S_{k+1}} - sum_{i>k} g_i w_i and dL/dsigma_k = delta_k dL/ds_k, in float64; it is scattered through the
level blend and the trilinear weights into the kept corners.  A midpoint outside the bounds or, given an occupancy
grid, in an empty macro cell (the kernel's fp32 cell lookup) gets no gradient, as in the kernel."""
import numpy as np

from grid_render_grad_ref import empty_cells
from grid_visibility_ref import corners

f32 = np.float32


def proposal_grad(levels, bounds, origins, directions, radii, t_samples, d_weights, occupancy=None, block=8,
                  chunk=512):
    """levels: [(density [nz, ny, nx] (0 at dropped points), index [nz, ny, nx] (SH row or -1))] -> per level the
    gradient [M_l] float64 in SH-row order."""
    lo32, hi32 = np.asarray(bounds[0], f32), np.asarray(bounds[1], f32)
    L = len(levels)
    dens = [np.asarray(d, np.float64).reshape(-1) for d, _ in levels]
    index = [np.asarray(i).reshape(-1) for _, i in levels]
    shapes = [np.asarray(d).shape[::-1] for d, _ in levels]  # (nx, ny, nz)
    out = [np.zeros(int((i >= 0).sum())) for i in index]
    s0 = np.max((hi32 - lo32) / (np.array(shapes[0]) - 1).astype(f32))  # fp32, as the kernel's s0_max
    o32, d32 = np.asarray(origins, f32).reshape(-1, 3), np.asarray(directions, f32).reshape(-1, 3)
    rad = np.asarray(radii, f32).reshape(-1)
    t = np.asarray(t_samples, f32)
    g = np.asarray(d_weights, np.float64)
    B = t.shape[0]
    dn = np.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2])
    for c0 in range(0, B, chunk):
        sl = slice(c0, min(B, c0 + chunk))
        with np.errstate(over="ignore", invalid="ignore"):
            tm = (t[sl, :-1] + t[sl, 1:]) * f32(0.5)
            delta = ((t[sl, 1:] - t[sl, :-1]) * dn[sl, None]).astype(np.float64)
            x32 = o32[sl, None, :] + tm[..., None] * d32[sl, None, :]
        live = np.all((x32 >= lo32) & (x32 <= hi32), axis=-1)
        x32 = np.where(live[..., None], x32, lo32)  # outside: any in-range lattice position, weighted 0 below
        if occupancy is not None:
            live &= ~empty_cells(occupancy, block, np.array(shapes[0]), bounds, x32)
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.log2(f32(np.sqrt(3.0)) * rad[sl, None] * tm / s0)
        lam = np.clip(np.nan_to_num(lam, nan=0.0, neginf=0.0, posinf=L - 1), f32(0), f32(L - 1))
        a = np.minimum(np.floor(lam).astype(np.int64), L - 1)
        f = np.where(a == L - 1, 0.0, (lam - a.astype(f32)).astype(np.float64))
        wl = [np.where(a == lvl, 1 - f, 0.0) + np.where(a + 1 == lvl, f, 0.0) for lvl in range(L)]
        cs = [corners(shapes[lvl], lo32, hi32, x32) for lvl in range(L)]
        sigma = sum(wl[lvl] * sum(w * dens[lvl][p] for p, w in cs[lvl]) for lvl in range(L))
        s = np.where(live, sigma, 0.0) * delta
        S_after = np.cumsum(s, axis=1)
        S_before = S_after - s
        w = np.exp(-S_before) - np.exp(-S_after)
        gw = g[sl] * w
        suffix = np.cumsum(gw[:, ::-1], axis=1)[:, ::-1] - gw  # sum_{i>k} g_i w_i
        d_sigma = np.where(live, delta * (g[sl] * np.exp(-S_after) - suffix), 0.0)
        for lvl in range(L):
            for p, wc in cs[lvl]:
                row = index[lvl][p]
                sel = live & (row >= 0) & (wl[lvl] > 0)
                np.add.at(out[lvl], row[sel], (d_sigma * wl[lvl] * wc)[sel])
    return out
