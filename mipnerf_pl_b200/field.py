"""Looking at the geometry of a trained field: density on a 3D lattice and its isosurface as a mesh.

* `MipNerf.query_density` evaluates the density at Gaussians (means, diagonal covariances); on the tensor cores it is
  the density-only mode of the level kernel (IPE -> trunk -> density head, nothing else).
* `density_grid` queries a lattice in z-slabs.  By default each lattice point is the Gaussian of its voxel (variance
  step**2 / 12 per axis, a uniform voxel's), so the IPE integrates the field over the voxel's footprint and the grid is
  anti-aliased at its own scale.
* `isosurface` extracts the `grid > iso` surface with the library's marching-tetrahedra kernels, and optionally vertex
  normals from the grid's gradient; `extract_mesh` is both.
* `mesh_colors` colours vertices with `MipNerf.query_radiance` (the radiance mode of the level kernel on the tensor
  cores), each vertex seen along its inward normal; `extract_mesh(colors=True)` adds normals and colours.
* `MipNerf.query_radiance_dirs` / `query_radiance_proj` see every point from one shared set of directions (the trunk
  once per point, the view layer's ReLU and the colour head per direction); `bake_sh` projects that colour onto real
  spherical harmonics over `sphere_quadrature`, `mesh_sh` does so at mesh vertices, and `eval_sh` evaluates the result.
* `write_ply` writes a binary PLY (optionally with normals and colours) with no dependency.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _cabi
from .ops import _call, _dev, _f32

DEFAULT_BOUNDS = ((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))
Resolution = Union[int, Sequence[int]]


def _resolution(resolution: Resolution) -> Tuple[int, int, int]:
    """(nx, ny, nz)."""
    res = (int(resolution),) * 3 if isinstance(resolution, (int, np.integer)) else tuple(int(r) for r in resolution)
    if len(res) != 3 or min(res) < 2:
        raise ValueError(f"resolution {resolution!r}: need an int or (nx, ny, nz), each >= 2")
    return res


def lattice_axes(resolution: Resolution, bounds=DEFAULT_BOUNDS, device="cuda"):
    """The lattice coordinates per axis, fp32: lo[a] + idx * step[a] with step[a] = (hi[a] - lo[a]) / (n[a] - 1), each
    operation rounded to fp32 (the positions the isosurface kernels give the lattice points)."""
    n = _resolution(resolution)
    lo = np.asarray(bounds[0], dtype=np.float32)
    hi = np.asarray(bounds[1], dtype=np.float32)
    step = (hi - lo) / (np.asarray(n, dtype=np.float32) - np.float32(1))
    axes = [torch.arange(n[a], dtype=torch.float32, device=device) * float(step[a]) + float(lo[a]) for a in range(3)]
    return axes, step


@torch.no_grad()
def density_grid(model, resolution: Resolution, bounds=DEFAULT_BOUNDS, variance=None,
                 slab_points: int = 1 << 22, z_range: Optional[Tuple[int, int]] = None) -> torch.Tensor:
    """Density (softplus(raw + density_bias)) of `model` on a lattice -> [nz, ny, nx] on the model's device.  Point
    (i, j, k) sits at lo + (i, j, k) * step; `variance` (a float or one per axis) is the diagonal covariance of every
    query, by default step**2 / 12 per axis; 0 gives a point-sampled grid.  Queried in z-slabs of at most
    `slab_points` points, so that the memory beyond the grid stays bounded.  `z_range` (z0, z1): only lattice layers
    [z0, z1), as [z1 - z0, ny, nx], equal bit for bit to those rows of the whole grid (the points are the same and
    the queries do not depend on how the points are batched).  Under no_grad: no graph, even on an autograd model."""
    dev = next(model.parameters()).device
    nx, ny, nz = _resolution(resolution)
    z0, z1 = (0, nz) if z_range is None else (int(z_range[0]), int(z_range[1]))
    if not 0 <= z0 <= z1 <= nz:
        raise ValueError(f"z_range {z_range!r}: need 0 <= z0 <= z1 <= nz = {nz}")
    (xs, ys, zs), step = lattice_axes((nx, ny, nz), bounds, dev)
    var = step.astype(np.float32) ** 2 / np.float32(12) if variance is None else np.broadcast_to(
        np.asarray(variance, dtype=np.float32), (3,))
    covs_row = torch.tensor(np.asarray(var, dtype=np.float32), device=dev)
    out = torch.empty(z1 - z0, ny, nx, device=dev)
    slab = max(1, slab_points // (nx * ny))
    yy, xx = torch.meshgrid(ys, xs, indexing="ij")
    for s in range(z0, z1, slab):
        z = zs[s:min(s + slab, z1)]
        means = torch.stack([xx.expand(len(z), ny, nx), yy.expand(len(z), ny, nx),
                             z[:, None, None].expand(len(z), ny, nx)], dim=-1)
        covs = covs_row.expand(len(z), ny, nx, 3)
        out[s - z0:s - z0 + len(z)] = model.query_density(means, covs)
    return out


def isosurface(grid: torch.Tensor, iso: float, bounds=DEFAULT_BOUNDS, normals: bool = False):
    """The surface `grid > iso` of a [nz, ny, nx] grid whose lattice spans `bounds` -> (verts [V,3] fp32, faces [F,3]
    int32) on the grid's device.  Marching tetrahedra (6 per cell): a watertight, consistently oriented mesh whose
    normals point from inside (> iso) to outside; NaN counts as outside.  Bit-reproducible.  With `normals`, also the
    unit vertex normals [V,3] from the grid's gradient (central differences, interpolated along each vertex's edge),
    pointing outside; (0, 0, 0) where the gradient is zero or not finite: (verts, faces, normals)."""
    dev = _dev(grid)
    if grid.dim() != 3:
        raise ValueError(f"grid must be [nz, ny, nx], got {tuple(grid.shape)}")
    g = _f32(grid)
    nz, ny, nx = g.shape
    lib = _cabi.lib()
    nbytes = lib.mipnerf_b200_isosurface_scratch_bytes(nx, ny, nz)
    if nbytes == 0:
        raise ValueError(f"grid {tuple(grid.shape)}: need at least 2 points per axis")
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    lo = (C.c_float * 3)(*[float(v) for v in bounds[0]])
    hi = (C.c_float * 3)(*[float(v) for v in bounds[1]])
    _call(dev, "isosurface", lib.mipnerf_b200_isosurface_count, g.data_ptr(), nx, ny, nz, float(iso),
          scratch.data_ptr(), nbytes, counts.data_ptr())
    nv, nf = (int(v) for v in counts.tolist())
    verts = torch.empty(nv, 3, device=dev)
    faces = torch.empty(nf, 3, dtype=torch.int32, device=dev)
    _call(dev, "isosurface", lib.mipnerf_b200_isosurface_emit, g.data_ptr(), nx, ny, nz, lo, hi, float(iso),
          scratch.data_ptr(), verts.data_ptr() if nv else None, faces.data_ptr() if nf else None)
    if not normals:
        return verts, faces
    nrm = torch.empty(nv, 3, device=dev)
    _call(dev, "isosurface", lib.mipnerf_b200_isosurface_normals, g.data_ptr(), nx, ny, nz, lo, hi, float(iso),
          scratch.data_ptr(), nrm.data_ptr() if nv else None)
    return verts, faces, nrm


@torch.no_grad()
def mesh_colors(model, verts: torch.Tensor, normals: torch.Tensor, variance, slab_points: int = 1 << 22) -> torch.Tensor:
    """The colour [V,3] of `model` at mesh vertices: the radiance (`MipNerf.query_radiance`) of each vertex's Gaussian
    (diagonal `variance`, a float or one per axis, e.g. the voxel's step**2 / 12) seen along -normal, a ray arriving at
    the surface from outside.  Queried in chunks of at most `slab_points` vertices, under no_grad."""
    dev = next(model.parameters()).device
    v = _f32(verts).to(dev).reshape(-1, 3)
    d = -_f32(normals).to(dev).reshape(-1, 3)
    var = torch.tensor(np.broadcast_to(np.asarray(variance, dtype=np.float32), (3,)).copy(), device=dev)
    out = torch.empty(v.shape[0], 3, device=dev)
    for o in range(0, v.shape[0], slab_points):
        vv = v[o:o + slab_points]
        out[o:o + len(vv)] = model.query_radiance(vv, var.expand(len(vv), 3), d[o:o + slab_points])[0]
    return out


# Real spherical harmonics up to degree 3 in the convention of the common `eval_sh` (PlenOctrees / Plenoxels / 3D
# Gaussian splatting): basis k = l^2 + l + m, orthonormal on the unit sphere, with these constants and signs.
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)
SH_MAX_DEGREE = 3


def _sh_terms(x, y, z, degree: int):
    """The (degree + 1)^2 basis functions at (x, y, z), as a list (numpy or torch arithmetic alike)."""
    if not 0 <= int(degree) <= SH_MAX_DEGREE:
        raise ValueError(f"degree {degree}: need 0..{SH_MAX_DEGREE}")
    out = [SH_C0 + 0 * x]
    if degree >= 1:
        out += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if degree >= 2:
        xx, yy, zz = x * x, y * y, z * z
        out += [SH_C2[0] * x * y, SH_C2[1] * y * z, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * x * z,
                SH_C2[4] * (xx - yy)]
    if degree >= 3:
        out += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * x * y * z, SH_C3[2] * y * (4 * zz - xx - yy),
                SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy),
                SH_C3[5] * z * (xx - yy), SH_C3[6] * x * (xx - 3 * yy)]
    return out


def sh_basis(dirs, degree: int) -> np.ndarray:
    """Real SH basis [..., (degree + 1)^2] at unit directions dirs [..., 3], float64 on the host; degree 0..3, the
    `eval_sh` convention (SH_C0 = 0.28209479..., Y_1 = -C1 y, Y_2 = C1 z, Y_3 = -C1 x, ...)."""
    d = np.asarray(torch.as_tensor(dirs).detach().cpu().numpy() if isinstance(dirs, torch.Tensor) else dirs,
                   dtype=np.float64)
    if d.shape[-1] != 3:
        raise ValueError(f"dirs {d.shape}: need [..., 3]")
    return np.stack(_sh_terms(d[..., 0], d[..., 1], d[..., 2], degree), axis=-1)


def sh_degree(num_coeffs: int) -> int:
    """The degree of an expansion with num_coeffs = (degree + 1)^2 coefficients."""
    deg = int(round(num_coeffs ** 0.5)) - 1
    if (deg + 1) ** 2 != num_coeffs or not 0 <= deg <= SH_MAX_DEGREE:
        raise ValueError(f"{num_coeffs} coefficients: need (degree + 1)^2 with degree 0..{SH_MAX_DEGREE}")
    return deg


def eval_sh(coeffs: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """The colour of an SH expansion: coeffs [..., K, C] with K = (degree + 1)^2, dirs [..., 3] (unit; broadcast against
    coeffs' leading dimensions) -> [..., C] = sum_k Y_k(dir) coeffs[..., k, :], in coeffs' dtype and device.  No
    activation: a bake of activated colours evaluates to colours."""
    deg = sh_degree(coeffs.shape[-2])
    d = dirs.to(device=coeffs.device, dtype=coeffs.dtype)
    y = torch.stack(_sh_terms(d[..., 0], d[..., 1], d[..., 2], deg), dim=-1)
    return (y.unsqueeze(-1) * coeffs).sum(dim=-2)


def sphere_quadrature(n_theta: int, n_phi: Optional[int] = None):
    """A quadrature on the unit sphere: Gauss-Legendre in cos(theta) (n_theta nodes) times n_phi uniform azimuths
    (default 2 n_theta, offset by half a step) -> (dirs [n_theta n_phi, 3], weights [n_theta n_phi]), float64 on the host,
    weights summing to 4 pi.  Exact for every product of two spherical harmonics of degree <= n_theta - 1, so that SH
    projections up to that degree are exact for band-limited functions."""
    n_theta = int(n_theta)
    n_phi = 2 * n_theta if n_phi is None else int(n_phi)
    if n_theta < 1 or n_phi < 1:
        raise ValueError(f"n_theta {n_theta}, n_phi {n_phi}: need >= 1")
    z, wz = np.polynomial.legendre.leggauss(n_theta)
    phi = 2.0 * np.pi * (np.arange(n_phi) + 0.5) / n_phi
    zz, pp = np.meshgrid(z, phi, indexing="ij")
    r = np.sqrt(np.maximum(0.0, 1.0 - zz * zz))
    dirs = np.stack([r * np.cos(pp), r * np.sin(pp), zz], axis=-1).reshape(-1, 3)
    weights = (wz[:, None] * np.full(n_phi, 2.0 * np.pi / n_phi)[None, :]).reshape(-1)
    return dirs, weights


def sh_table(degree: int, n_theta: int):
    """The projection of `bake_sh`: (dirs [D, 3] float64, table [D, K] float64 = w_d Y_k(dir_d)) of
    sphere_quadrature(n_theta)."""
    if not 0 <= int(degree) <= min(SH_MAX_DEGREE, int(n_theta) - 1):
        raise ValueError(f"degree {degree} with n_theta {n_theta}: need 0 <= degree <= min(3, n_theta - 1)")
    dirs, w = sphere_quadrature(n_theta)
    return dirs, w[:, None] * sh_basis(dirs, degree)


@torch.no_grad()
def bake_sh(model, means: torch.Tensor, covs: Optional[torch.Tensor] = None, degree: int = 2, n_theta: int = 8,
            raw: bool = False) -> torch.Tensor:
    """The view-dependent colour of `model` at Gaussians as real SH coefficients [..., (degree + 1)^2, 3] (`eval_sh`
    convention, degree 0..3): coeffs_k = sum_d w_d Y_k(d) rgb(d) over sphere_quadrature(n_theta) (n_theta * 2 n_theta
    directions; the default 8 gives 128), i.e. the L2 projection of the colour onto the basis, in one
    `MipNerf.query_radiance_proj` call (the table w_d Y_k(d) built in float64 and rounded to fp32; no [..., D, 3] colour
    array).  `raw`: the raw colour head instead of the activated colour.  Under no_grad."""
    dirs, table = sh_table(degree, n_theta)
    dev = means.device
    d32 = torch.tensor(dirs, dtype=torch.float32, device=dev)
    t32 = torch.tensor(table, dtype=torch.float32, device=dev)
    return model.query_radiance_proj(means, covs, d32, t32, raw=raw)[0]


@torch.no_grad()
def mesh_sh(model, verts: torch.Tensor, variance, degree: int = 2, n_theta: int = 8,
            slab_points: int = 1 << 22) -> torch.Tensor:
    """The view-dependent colour [V, (degree + 1)^2, 3] of `model` at mesh vertices as SH coefficients (`bake_sh` of each
    vertex's Gaussian, diagonal `variance`, a float or one per axis, e.g. the voxel's step**2 / 12): the counterpart
    of `mesh_colors` for every direction at once.  Queried in chunks of at most `slab_points` vertices, under no_grad."""
    dev = next(model.parameters()).device
    v = _f32(verts).to(dev).reshape(-1, 3)
    var = torch.tensor(np.broadcast_to(np.asarray(variance, dtype=np.float32), (3,)).copy(), device=dev)
    out = torch.empty(v.shape[0], (int(degree) + 1) ** 2, 3, device=dev)
    for o in range(0, v.shape[0], slab_points):
        vv = v[o:o + slab_points]
        out[o:o + len(vv)] = bake_sh(model, vv, var.expand(len(vv), 3), degree, n_theta)
    return out


def voxel_variance(resolution: Resolution, bounds=DEFAULT_BOUNDS) -> np.ndarray:
    """step**2 / 12 per axis: the variance of a uniform voxel of the lattice (density_grid's default)."""
    _, step = lattice_axes(resolution, bounds, "cpu")
    return step.astype(np.float32) ** 2 / np.float32(12)


def extract_mesh(model, threshold: float, resolution: Resolution = 256, bounds=DEFAULT_BOUNDS,
                 variance=None, colors: bool = False):
    """The surface density > threshold of `model` inside `bounds` -> (verts, faces) on the model's device.  With
    `colors`: (verts, faces, normals, colors), the normals from the density grid's gradient and the colours from
    `mesh_colors` with the grid's variance (by default the voxel's, step**2 / 12)."""
    grid = density_grid(model, resolution, bounds, variance)
    if not colors:
        return isosurface(grid, threshold, bounds)
    verts, faces, normals = isosurface(grid, threshold, bounds, normals=True)
    var = voxel_variance(resolution, bounds) if variance is None else variance
    return verts, faces, normals, mesh_colors(model, verts, normals, var)


def write_ply(path: str, verts, faces, colors=None, normals=None) -> None:
    """Binary little-endian PLY: float x, y, z per vertex, then (with `normals`) float nx, ny, nz and (with `colors`,
    [V,3] in [0, 1]) uchar red, green, blue = round(255 clamp(c, 0, 1)); uchar-counted int vertex_indices per face."""
    v = np.ascontiguousarray(torch.as_tensor(verts).detach().cpu().numpy(), dtype="<f4").reshape(-1, 3)
    f = np.ascontiguousarray(torch.as_tensor(faces).detach().cpu().numpy(), dtype="<i4").reshape(-1, 3)
    rec = np.empty(len(f), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    rec["n"] = 3
    rec["idx"] = f
    fields = [("xyz", "<f4", (3,))]
    props = "property float x\nproperty float y\nproperty float z\n"
    if normals is not None:
        fields.append(("n", "<f4", (3,)))
        props += "property float nx\nproperty float ny\nproperty float nz\n"
    if colors is not None:
        fields.append(("rgb", "u1", (3,)))
        props += "property uchar red\nproperty uchar green\nproperty uchar blue\n"
    vert = np.empty(len(v), dtype=fields)
    vert["xyz"] = v
    if normals is not None:
        vert["n"] = np.asarray(torch.as_tensor(normals).detach().cpu().numpy(), dtype=np.float32).reshape(-1, 3)
    if colors is not None:
        c = np.asarray(torch.as_tensor(colors).detach().float().cpu().numpy(), dtype=np.float32).reshape(-1, 3)
        vert["rgb"] = np.round(np.clip(c, 0.0, 1.0) * np.float32(255)).astype(np.uint8)
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(v)}\n{props}"
              f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(rec.tobytes())
