"""numpy implementation of the vertex-normal rule of mipnerf_b200_isosurface_normals, in the vertex order of
isosurface_ref.isosurface: the grid gradient at both ends of each vertex's edge (central differences over 2 step per
axis, one-sided over step at the box faces), interpolated with the vertex's t, negated and normalised; (0, 0, 0) where
that is zero or not finite.  Every operation is a float32 one, as the kernel's explicitly rounded ones."""
import numpy as np

import isosurface_ref as R


def gradient(grid, step):
    """[nz, ny, nx, 3] float32 (d/dx, d/dy, d/dz) of a [nz, ny, nx] grid."""
    g = np.asarray(grid, dtype=np.float32)
    out = np.empty(g.shape + (3,), dtype=np.float32)
    for a in range(3):
        ax = 2 - a  # x is the last array axis
        n = g.shape[ax]
        s = np.float32(step[a])
        idx = np.arange(n)
        plus = np.take(g, np.minimum(idx + 1, n - 1), axis=ax)
        minus = np.take(g, np.maximum(idx - 1, 0), axis=ax)
        shape = [1, 1, 1]
        shape[ax] = n
        edge = ((idx == 0) | (idx == n - 1)).reshape(shape)
        den = np.where(edge, s, np.float32(2) * s).astype(np.float32)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            out[..., a] = ((plus - minus).astype(np.float32) / den).astype(np.float32)
    return out


def normals(grid, iso, bounds):
    """(verts, faces, normals [V,3] float32) of isosurface_ref.isosurface(grid, iso, bounds)."""
    g = np.asarray(grid, dtype=np.float32)
    verts, faces, edges = R.isosurface(g, iso, bounds)
    nz, ny, nx = g.shape
    lo = np.asarray(bounds[0], dtype=np.float32)
    hi = np.asarray(bounds[1], dtype=np.float32)
    step = (hi - lo) / (np.array([nx, ny, nz]).astype(np.float32) - np.float32(1))
    grad = gradient(g, step)
    a, b = edges[:, 0], edges[:, 1]  # lattice (i, j, k) of the two ends
    va, vb = g[a[:, 2], a[:, 1], a[:, 0]], g[b[:, 2], b[:, 1], b[:, 0]]
    iso = np.float32(iso)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        t = ((iso - va).astype(np.float32) / (vb - va).astype(np.float32)).astype(np.float32)
        t = np.where(np.isnan(t), np.float32(0.5), t).astype(np.float32)
        ga, gb = grad[a[:, 2], a[:, 1], a[:, 0]], grad[b[:, 2], b[:, 1], b[:, 0]]
        n = (ga + t[:, None] * (gb - ga).astype(np.float32)).astype(np.float32)
        sq = n * n
        length = np.sqrt((sq[:, 0] + sq[:, 1]).astype(np.float32) + sq[:, 2]).astype(np.float32)
        ok = (length > 0) & np.isfinite(length)
        out = np.where(ok[:, None], (-n / np.where(ok, length, np.float32(1))[:, None]).astype(np.float32),
                       np.float32(0))
    return verts, faces, out.astype(np.float32)


def face_normals(verts, faces):
    """Area-weighted face normals summed per vertex, [V,3] float64 (the faces' orientation)."""
    v = np.asarray(verts, dtype=np.float64)
    fn = np.cross(v[faces[:, 1]] - v[faces[:, 0]], v[faces[:, 2]] - v[faces[:, 0]])
    acc = np.zeros_like(v)
    for k in range(3):
        np.add.at(acc, faces[:, k], fn)
    return acc
