"""float64 torch restatement of the total-variation prior of a baked grid (mipnerf_b200_grid_tv,
BakedGrid.total_variation), differentiable in each level's parameters: the kept points' densities [M_l] in SH-row order
and their SH rows [M_l, (degree + 1)^2, 3].  Gradients come from autograd on it.

Per level, on its own lattice: for each kept point p and axis a, q = p + e_a.  D_a sigma(p) = sigma(q) - sigma(p), a
dropped q reading 0; D_a c(p) = c(q) - c(p) where q is kept and 0 where it is dropped; both 0 where q lies outside the
lattice.  Per point, sqrt(eps + sum_a (D_a sigma)^2) and sum_{k,ch} sqrt(eps + sum_a (D_a c_{k,ch})^2); TV_density and
TV_sh are their sums over all levels' kept points divided by M, the number of kept points (0 when M = 0)."""
import numpy as np
import torch

from mipnerf_pl_b200.baked import TV_EPS


def level_terms(kept_density, sh, index, eps=TV_EPS):
    """(density terms [M], SH terms [M]) of one level: kept_density [M] and sh [M, nc, 3] float64 in SH-row order,
    index [nz, ny, nx] (the SH row of each lattice point, -1 where dropped)."""
    idx = torch.as_tensor(np.asarray(index), dtype=torch.int64)
    m = int((idx >= 0).sum())
    if m == 0:
        return kept_density.new_zeros(0), kept_density.new_zeros(0)
    rows = sh.reshape(m, -1)
    n = idx.shape  # (nz, ny, nx)
    kz, ky, kx = (idx >= 0).nonzero(as_tuple=True)
    order = torch.argsort(idx[kz, ky, kx])
    pz, py, px = kz[order], ky[order], kx[order]  # lattice position of row r
    d_sigma, d_c = [], []
    for dz, dy, dx in ((0, 0, 1), (0, 1, 0), (1, 0, 0)):  # axes x, y, z
        qz, qy, qx = pz + dz, py + dy, px + dx
        inside = (qz < n[0]) & (qy < n[1]) & (qx < n[2])
        qi = torch.where(inside, idx[qz.clamp(max=n[0] - 1), qy.clamp(max=n[1] - 1), qx.clamp(max=n[2] - 1)],
                         torch.full_like(qz, -1))
        kept_q = qi >= 0
        sigma_q = torch.where(kept_q, kept_density[qi.clamp(min=0)], torch.zeros((), dtype=torch.float64))
        d_sigma.append(torch.where(inside, sigma_q - kept_density, torch.zeros((), dtype=torch.float64)))
        d_c.append(torch.where(kept_q[:, None], rows[qi.clamp(min=0)] - rows, torch.zeros((), dtype=torch.float64)))
    t_sigma = torch.sqrt(eps + sum(d * d for d in d_sigma))
    t_sh = torch.sqrt(eps + sum(d * d for d in d_c)).sum(dim=1)
    return t_sigma, t_sh


def total_variation(params, indices, eps=TV_EPS):
    """(TV_density, TV_sh, per-level terms) of params [(kept_density, sh) per level] and indices [index per level]."""
    terms = [level_terms(kd, sh, i, eps) for (kd, sh), i in zip(params, indices)]
    m = sum(t[0].numel() for t in terms)
    if m == 0:
        zero = torch.zeros((), dtype=torch.float64)
        return zero, zero, terms
    return sum(t[0].sum() for t in terms) / m, sum(t[1].sum() for t in terms) / m, terms
