"""Baked grids: the field sampled once on a mip pyramid of lattices (density and raw spherical-harmonic colour), and
frames rendered from it by a CUDA ray marcher instead of the MLP.

* Level l of `levels` has n_l = (n_0 - 1) / 2^l + 1 points per axis over the same bounds, so the lattices nest.  Its
  density is `field.density_grid` with the default voxel variance (step_l^2 / 12 per axis): the IPE integrates the
  field over each voxel, so level l is the field pre-filtered at 2^l times the finest scale, not a subsampled copy.
* A point is kept where the 3x3x3 dilation of `density > threshold` holds; elsewhere the baked density is 0 (a dropped
  point's density is at most `threshold`).  The kept points' colour is `field.bake_sh(raw=True)` of their voxel
  Gaussians, stored fp32 [M_l, (degree + 1)^2, 3]; the renderer applies the model's activation after the SH sum.
* The occupancy grid marks macro cells of `block`^3 finest cells.  A cell is empty only if every level's baked
  density is 0 on the cell's lattice points widened by one point of that level, so that every position in the cell
  (and any position a rounding error outside it) interpolates to exactly 0 at every level: skipping empty cells
  leaves the rendered result bit for bit unchanged.
* Memory layout read by csrc/grid_render.cu, decided here and there only.  Each lattice point has one 8-byte word
  (density bits, SH row or -1), and the SH rows are in the order of the kept points (x fastest).  A dense grid holds
  the words of level l as one int32 [nz, ny, nx, 2] array, x fastest.  A sparse grid (`sparsify`) holds them in
  bricks of 8^3 points: an int32 table [tz, ty, tx] (t = ceil(n / 8) per axis) of brick ids in raster order (x
  fastest), -1 for a brick not stored, and an int32 pool [num_bricks, 8, 8, 8, 2]; point (i, j, k) is point (k & 7, j &
  7, i & 7) of brick (k >> 3, j >> 3, i >> 3).  A brick is stored iff one of its points inside the lattice holds a word
  other than (+0.0 bits, -1), and points past the lattice in an edge brick hold (0, -1), so an absent brick reads
  what the dense array holds there: the encoding is lossless and renders bit for bit as the dense grid.  The rule
  looks at rows as well as densities because a kept point may have density 0 (the keep mask is a dilation, and
  fine-tuning projects onto >= 0) and the renderer still adds its colour wherever the blended density is non-zero.

The renderer (`BakedGrid.render`, `render_baked_frame`) marches K = max(1, ceil((far - near) |d| / step)) samples at
t_k = near + (k + 1/2) dt, blends two levels picked by the cone footprint (lambda = log2(sqrt(3) radii t / s_0)) and
composites as `volumetric_rendering`, stopping once the transmittance drops below 1e-4 (include/mipnerf_b200.h).

Pruning (`BakedGrid.visibility`, `BakedGrid.prune`, `prune_grid`) drops the kept points that no training ray sees: per
kept point the largest blending weight T_k alpha_k, times the coefficient the renderer gives its colour, over every
training ray (PlenOctrees), and a threshold on it.

Quantization (`BakedGrid.quantize`, SNeRG's 8-bit storage) stores the SH rows as uint8 with an affine code per level,
coefficient and channel: offset = the column's minimum, scale = (max - min) / 255 in fp32, q = clamp(round((c - offset) /
scale), 0, 255) (0 for a constant column).  A coefficient reads as deq(q) = fl32(fl32(q * scale) + offset), two
explicitly rounded fp32 operations, in `dequantize` and in the renderer's kernel alike
(mipnerf_b200_grid_render_u8), so a quantized grid renders bit for bit as its `dequantize()` does.  The intended
pipeline is bake -> prune -> fine-tune -> quantize: a quantized grid is not pruned or trained.

Sparse cells (`BakedGrid.sparsify`, the occupied blocks PlenOctrees and SNeRG store) keep only the non-empty bricks
of each level, fp32 or quantized rows alike; `densify` restores the dense grid bit for bit.  A sparse grid is a
viewer format, the last step of bake -> prune -> fine-tune -> quantize -> sparsify: it renders
(mipnerf_b200_grid_render_bricks) and saves, and is not pruned, trained or (de)quantized.

Streamed bakes (`bake_grid(sparse=True)`, `sparse_grid_structure`) write the sparse layout directly, walking each
level in z-slabs of brick layers, so that a bake at 1025^3 or 2049^3 never holds a level's whole lattice; the result
equals the dense bake followed by `sparsify()` in every array.  `bake_grid(prune=bank)` prunes inside the bake: the
visibility runs on the structure (cells and occupancy, on the bricks with `sparse`) before any SH row exists, so only
the surviving points' rows are baked; the result equals `prune_grid` of the unpruned bake, then `quantize` and
`sparsify`.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _cabi
from .field import DEFAULT_BOUNDS, Resolution, _resolution, bake_sh, density_grid, lattice_axes, voxel_variance
from .ops import _call, _dev, _f32, _rays_struct
from .rays import BLENDER_CAMERA_ANGLE_X, Rays
from .render import gather_rows, generate_rays, shard_rows

MAX_LEVELS = _cabi.GRID_MAX_LEVELS
DEFAULT_BLOCK = 8
DEFAULT_THRESHOLD = 1e-2
# finetune_grid's Adam learning rates (README, "Fine-tuning a baked grid")
FINETUNE_LR_DENSITY = 0.1
FINETUNE_LR_SH = 0.01
# prune_grid's visibility threshold (README, "Pruning a baked grid by visibility")
DEFAULT_WEIGHT_THRESHOLD = 1e-5
# the epsilon inside every square root of BakedGrid.total_variation: it keeps the gradient finite where a point's
# differences are all 0, and adds sqrt(TV_EPS) per point and term, far below any difference a grid resolves
TV_EPS = 1e-8
_FORMAT = 1
_FORMAT_U8 = 2  # a quantized grid: uint8 SH rows plus per-level scale / offset
_FORMAT_BRICKS = 3  # a sparse grid: per-level brick table and pool, fp32 or uint8 rows
BRICK = 8  # brick edge in lattice points, every level
_SLAB_BYTES = 1 << 28  # sparsify / densify: bytes of dense cells handled at once


def level_resolutions(resolution: Resolution, levels: int) -> List[Tuple[int, int, int]]:
    """(nx, ny, nz) of every level: (n_0 - 1) / 2^l + 1 per axis."""
    n0 = _resolution(resolution)
    if not 1 <= int(levels) <= MAX_LEVELS:
        raise ValueError(f"levels {levels}: need 1..{MAX_LEVELS}")
    scale = 1 << (int(levels) - 1)
    if any((n - 1) % scale for n in n0):
        raise ValueError(f"resolution {n0}: n - 1 must be divisible by 2^(levels - 1) = {scale} on every axis")
    return [tuple((n - 1) // (1 << lvl) + 1 for n in n0) for lvl in range(int(levels))]


def _cell_matrix(n_cells: int, n_points: int, block: int, scale: int, device) -> torch.Tensor:
    """[n_cells, n_points] 0/1: the level points (spacing `scale` finest cells) macro cell I depends on, the points
    of finest cells [I block, (I + 1) block] widened by one point per side."""
    cell = torch.arange(n_cells, device=device)[:, None]
    p = torch.arange(n_points, device=device)[None, :]
    first = torch.div(cell * block, scale, rounding_mode="floor") - 1
    last = -torch.div(-(cell + 1) * block, scale, rounding_mode="floor") + 1
    return ((p >= first) & (p <= last)).to(torch.float32)


def _keep_mask(density: torch.Tensor, threshold: float) -> torch.Tensor:
    """The kept points of fp32 densities [nz, ny, nx]: the 3x3x3 dilation of density > threshold, nothing kept past
    the array's ends."""
    return torch.nn.functional.max_pool3d((density > threshold).to(torch.float32)[None, None], 3, 1, 1)[0, 0] > 0


def _occupancy_counts(nonzero: torch.Tensor, z0: int, nz: int, o, block: int, scale: int) -> torch.Tensor:
    """Per macro cell [oz, oy, ox] fp32, how many of the 0/1 points `nonzero` (lattice layers [z0, z0 + its depth) of a
    level of nz layers and point spacing `scale` finest cells) lie on the cell's lattice points widened by one point.
    Every count is an exact integer below 2^24, so `> 0` of a sum of such counts is exact."""
    dev = nonzero.device
    ax, ay = (_cell_matrix(o[2 - a], nonzero.shape[2 - a], block, scale, dev) for a in range(2))
    az = _cell_matrix(o[0], nz, block, scale, dev)[:, z0:z0 + nonzero.shape[0]]
    t = torch.einsum("kji,ai->kja", nonzero, ax)
    t = torch.einsum("kja,bj->kba", t, ay)
    return torch.einsum("kba,ck->cba", t, az)


@torch.no_grad()
def grid_structure(densities: Sequence[torch.Tensor], threshold: float, block: int = DEFAULT_BLOCK):
    """The mask, index and occupancy construction from the density grids of every level (no model; any device) ->
    (baked densities [nz, ny, nx] fp32, indices [nz, ny, nx] int32, occupancy [oz, oy, ox] uint8).  Level l keeps the
    3x3x3 dilation of density > threshold; its baked density is the density where kept and 0 elsewhere; its index is
    the row of a kept point among the level's kept points in x-fastest order and -1 elsewhere.  occupancy (o = ceil((n_0
    - 1) / block) per axis) is 0 only for macro cells whose widened lattice points have baked density 0 at every level."""
    if not 1 <= len(densities) <= MAX_LEVELS:
        raise ValueError(f"{len(densities)} levels: need 1..{MAX_LEVELS}")
    n0 = tuple(densities[0].shape)
    scale_max = 1 << (len(densities) - 1)
    if int(block) < 1 or int(block) % scale_max:
        raise ValueError(f"block {block}: need a positive multiple of 2^(levels - 1) = {scale_max}")
    if len(n0) != 3 or min(n0) < 2 or any((n - 1) % scale_max for n in n0):
        raise ValueError(f"level 0: grid {n0}, need [nz, ny, nx], each >= 2 with n - 1 divisible by {scale_max}")
    baked, indices = [], []
    dev = densities[0].device
    for lvl, dens in enumerate(densities):
        want = tuple((n - 1) // (1 << lvl) + 1 for n in n0)
        if tuple(dens.shape) != want:
            raise ValueError(f"level {lvl}: grid {tuple(dens.shape)}, need {want} nested in level 0's {n0}")
        d = dens.to(torch.float32)
        keep = _keep_mask(d, threshold)
        bd = torch.where(keep, d, torch.zeros((), device=dev))
        idx = torch.full(bd.shape, -1, dtype=torch.int32, device=dev)
        idx[keep] = torch.arange(int(keep.sum()), dtype=torch.int32, device=dev)
        baked.append(bd.contiguous())
        indices.append(idx)
    return baked, indices, grid_occupancy(baked, block)


@torch.no_grad()
def grid_occupancy(baked_densities: Sequence[torch.Tensor], block: int = DEFAULT_BLOCK) -> torch.Tensor:
    """The occupancy [oz, oy, ox] uint8 (o = ceil((n_0 - 1) / block) per axis) of nested baked density grids [nz, ny,
    nx] (level l: (n_0 - 1) / 2^l + 1 points per axis): 0 only for macro cells of `block`^3 finest cells whose lattice
    points, widened by one point of each level, have baked density 0 at every level."""
    n0 = tuple(baked_densities[0].shape)
    dev = baked_densities[0].device
    o = [-(-(n - 1) // block) for n in n0]  # (oz, oy, ox)
    occ = torch.zeros(o, dtype=torch.float32, device=dev)
    for lvl, bd in enumerate(baked_densities):
        occ += _occupancy_counts((bd != 0).to(torch.float32), 0, bd.shape[0], o, block, 1 << lvl)
    return (occ > 0).to(torch.uint8)


_MAX_ROWS = 2 ** 31 - 1  # SH row ids are int32


@torch.no_grad()
def sparse_grid_structure(density_fn, resolution: Resolution, levels: int = 1, threshold: float = DEFAULT_THRESHOLD,
                          block: int = DEFAULT_BLOCK, slab: Optional[int] = None):
    """`grid_structure` followed by the dense constructor and `sparsify()`, streamed: each level is walked in z-slabs
    of `slab` brick layers (lattice layers [8 z0, 8 z1); None: the whole level), so that no array the size of a
    level's lattice is ever held.  `density_fn(level, z0, z1)` returns that level's densities on lattice layers [z0,
    z1) as [z1 - z0, ny, nx] (level l of `level_resolutions(resolution, levels)`).  Returns (tables, pools, positions,
    occupancy): per level the int32 brick table and pool of `sparsify`, the int64 lattice positions (x fastest, z
    slowest) of the kept points in SH-row order, and the uint8 occupancy of `grid_occupancy`, every array bit for bit
    as the dense path gives it.  A level whose kept points would not fit int32 row ids is refused."""
    res = level_resolutions(resolution, levels)
    scale_max = 1 << (len(res) - 1)
    if int(block) < 1 or int(block) % scale_max:
        raise ValueError(f"block {block}: need a positive multiple of 2^(levels - 1) = {scale_max}")
    if slab is not None and int(slab) < 1:
        raise ValueError(f"slab {slab}: need >= 1 brick layer, or None for the whole level")
    o = tuple(-(-(n - 1) // int(block)) for n in res[0][::-1])
    occ = None
    tables, pools, positions = [], [], []
    for lvl, (nx, ny, nz) in enumerate(res):
        t = (-(-nz // BRICK), -(-ny // BRICK), -(-nx // BRICK))
        step = t[0] if slab is None else int(slab)
        tabs, bricks, pos = [], [], []
        rows = count = 0
        for b0 in range(0, t[0], step):
            b1 = min(b0 + step, t[0])
            z0, z1 = b0 * BRICK, min(b1 * BRICK, nz)
            # The halo: the keep mask's 3x3x3 dilation reads density > threshold one layer beyond the slab on each
            # side, clipped at the lattice ends (where max_pool3d's padding keeps nothing, as on the whole level).
            # The occupancy needs no halo: each slab adds its own points' counts to every macro cell whose widened
            # lattice points hold them, and the cell is occupied iff any slab's count is non-zero.
            h0, h1 = max(z0 - 1, 0), min(z1 + 1, nz)
            d = density_fn(lvl, h0, h1)
            if tuple(d.shape) != (h1 - h0, ny, nx):
                raise ValueError(f"density_fn({lvl}, {h0}, {h1}): shape {tuple(d.shape)}, need {(h1 - h0, ny, nx)}")
            d = d.to(torch.float32)
            keep = _keep_mask(d, threshold)[z0 - h0:z1 - h0]
            d = d[z0 - h0:z1 - h0]
            dev = d.device
            k = int(keep.sum())
            if rows + k > _MAX_ROWS:
                raise ValueError(f"level {lvl}: more than {_MAX_ROWS} kept points, beyond int32 SH row ids; use a "
                                 f"coarser resolution or a higher threshold")
            pos.append(keep.reshape(-1).nonzero().reshape(-1) + z0 * ny * nx)
            idx = torch.full(keep.shape, -1, dtype=torch.int32, device=dev)
            idx[keep] = torch.arange(rows, rows + k, dtype=torch.int32, device=dev)
            rows += k
            bd = torch.where(keep, d, torch.zeros((), device=dev))
            del d, keep
            counts = _occupancy_counts((bd != 0).to(torch.float32), z0, nz, o, int(block), 1 << lvl)
            occ = counts > 0 if occ is None else occ | (counts > 0)
            b = _brick_slab(torch.stack([bd.view(torch.int32), idx], dim=-1), 0, b1 - b0, t)
            del bd, idx
            tab, stored, count = _number_bricks(b, count)
            tabs.append(tab)
            # each slab's stored bricks stay a tensor of their own and are joined once per level: one copy per brick
            # and a transient of one pool, where growing one buffer by doubling copies up to twice and peaks at three
            # pools, and a count pass then a fill pass would query every density twice
            bricks.append(b[stored])
            del b
        tables.append(torch.cat(tabs))
        pools.append(torch.cat(bricks))
        del bricks
        positions.append(torch.cat(pos))
    return tables, pools, positions, occ.to(torch.uint8)


class BakedGrid:
    """A baked field: per level the density and SH index lattices and the SH rows, the bounds, the SH degree, the
    model's rgb_padding and the macro-cell occupancy.  `render` marches rays through it on the GPU; `save` / `load`
    keep it in one .npz.  With `sh_scale` and `sh_offset` (per level fp32 [(degree + 1)^2, 3]) the grid is quantized:
    `sh` holds uint8 rows read as fl(fl(q * scale) + offset) (`quantize`)."""

    def __init__(self, densities: Sequence[torch.Tensor], indices: Sequence[torch.Tensor], sh: Sequence[torch.Tensor],
                 occupancy: torch.Tensor, bounds=DEFAULT_BOUNDS, degree: int = 2, rgb_padding: float = 0.001,
                 block: int = DEFAULT_BLOCK, sh_scale: Optional[Sequence[torch.Tensor]] = None,
                 sh_offset: Optional[Sequence[torch.Tensor]] = None):
        cells = []
        for lvl, (d, i, c) in enumerate(zip(densities, indices, sh)):
            if d.shape != i.shape or d.dim() != 3:
                raise ValueError(f"level {lvl}: density {tuple(d.shape)}, index {tuple(i.shape)}, sh {tuple(c.shape)}")
            # (density bits, row) per lattice point: the kernel reads one 8-byte word per corner
            cells.append(torch.stack([_f32(d).view(torch.int32), i.to(torch.int32)], dim=-1).contiguous())
        self._setup((densities, indices, sh), "", cells, None, [tuple(c.shape[2::-1]) for c in cells], sh, occupancy,
                    bounds, degree, rgb_padding, block, sh_scale, sh_offset)

    @classmethod
    def from_bricks(cls, tables: Sequence[torch.Tensor], pools: Sequence[torch.Tensor],
                    resolutions: Sequence[Tuple[int, int, int]], sh: Sequence[torch.Tensor], occupancy: torch.Tensor,
                    bounds=DEFAULT_BOUNDS, degree: int = 2, rgb_padding: float = 0.001, block: int = DEFAULT_BLOCK,
                    sh_scale: Optional[Sequence[torch.Tensor]] = None,
                    sh_offset: Optional[Sequence[torch.Tensor]] = None) -> "BakedGrid":
        """A sparse grid from its bricks (the layout of `sparsify`): per level an int32 table [tz, ty, tx] (t = ceil(n
        / 8) of `resolutions[l]` = (nx, ny, nz)) and an int32 pool [num_bricks, 8, 8, 8, 2]; the other arguments as
        for the dense constructor.  Every table entry must be -1 or a brick id below num_bricks."""
        bricks, res = [], []
        for lvl, (t, p, r) in enumerate(zip(tables, pools, resolutions)):
            r = tuple(int(n) for n in r)
            want = tuple(-(-n // BRICK) for n in r[::-1])
            if len(r) != 3 or min(r) < 2 or t.dtype != torch.int32 or tuple(t.shape) != want:
                raise ValueError(f"level {lvl}: table {t.dtype} {tuple(t.shape)} for {r} points, need int32 {want}")
            if p.dtype != torch.int32 or p.dim() != 5 or tuple(p.shape[1:]) != (BRICK, BRICK, BRICK, 2):
                raise ValueError(f"level {lvl}: pool {p.dtype} {tuple(p.shape)}, need int32 [num_bricks, 8, 8, 8, 2]")
            if t.numel() and not (int(t.min()) >= -1 and int(t.max()) < p.shape[0]):
                raise ValueError(f"level {lvl}: table entries in [{int(t.min())}, {int(t.max())}], need -1 or a "
                                 f"brick id below {p.shape[0]}")
            bricks.append((t.contiguous(), p.contiguous()))
            res.append(r)
        grid = cls.__new__(cls)
        grid._setup((tables, pools, resolutions, sh), " of tables / pools / resolutions / sh", None, bricks, res, sh,
                    occupancy, bounds, degree, rgb_padding, block, sh_scale, sh_offset)
        return grid

    def _setup(self, per_level, names, cells, bricks, resolutions, sh, occupancy, bounds, degree,
               rgb_padding, block, sh_scale, sh_offset) -> None:
        """The constructors' shared part: `cells` (dense) or `bricks` (sparse, per level (table, pool)), one of them
        None, with the (nx, ny, nz) of each level; the per-level arguments `per_level` (`names`) need one count."""
        if not 0 <= int(degree) <= 3:
            raise ValueError(f"degree {degree}: need 0..3")
        counts = [len(a) for a in per_level]
        if len(set(counts)) != 1 or not 1 <= counts[0] <= MAX_LEVELS:
            raise ValueError(f"{' / '.join(map(str, counts))} levels{names}: need the same count, 1..{MAX_LEVELS}")
        self.degree = int(degree)
        self.rgb_padding = float(rgb_padding)
        self.block = int(block)
        self.bounds = (tuple(float(v) for v in bounds[0]), tuple(float(v) for v in bounds[1]))
        nc = (self.degree + 1) ** 2
        if (sh_scale is None) != (sh_offset is None):
            raise ValueError("sh_scale and sh_offset: give both (a quantized grid) or neither")
        quantized = sh_scale is not None
        if quantized and not (len(sh_scale) == len(sh_offset) == len(sh)):
            raise ValueError(f"{len(sh_scale)} / {len(sh_offset)} levels of sh_scale / sh_offset, {len(sh)} of sh")
        self.cells: Optional[List[torch.Tensor]] = cells  # dense: per level [nz, ny, nx, 2] int32
        self.bricks: Optional[List[Tuple[torch.Tensor, torch.Tensor]]] = bricks  # sparse: per level (table, pool)
        self._resolutions = [tuple(r) for r in resolutions]
        self.sh = []
        for lvl, c in enumerate(sh):
            if c.dim() != 3 or tuple(c.shape[1:]) != (nc, 3):
                raise ValueError(f"level {lvl}: sh {tuple(c.shape)}, need [M, {nc}, 3]")
            if quantized and c.dtype != torch.uint8:
                raise ValueError(f"level {lvl}: sh of a quantized grid must be uint8, got {c.dtype}")
            self.sh.append(c.detach().contiguous() if quantized else _f32(c))
        self.sh_scale: Optional[List[torch.Tensor]] = None  # quantized: per level fp32 [nc, 3]
        self.sh_offset: Optional[List[torch.Tensor]] = None
        if quantized:
            self.sh_scale, self.sh_offset = [], []
            for lvl, (s, o) in enumerate(zip(sh_scale, sh_offset)):
                s, o = _f32(s).to(self.device), _f32(o).to(self.device)
                if tuple(s.shape) != (nc, 3) or tuple(o.shape) != (nc, 3):
                    raise ValueError(f"level {lvl}: sh_scale {tuple(s.shape)}, sh_offset {tuple(o.shape)}, need {(nc, 3)}")
                if not bool(torch.isfinite(s).all() and torch.isfinite(o).all()):
                    raise ValueError(f"level {lvl}: sh_scale / sh_offset is not finite")
                self.sh_scale.append(s)
                self.sh_offset.append(o)
            # the tables as the kernel takes them by value ([MAX_LEVELS][16][3] fp32), copied to the host once
            self._deq_host = []
            for tabs in (self.sh_scale, self.sh_offset):
                pad = np.zeros((MAX_LEVELS, 16, 3), dtype=np.float32)
                for lvl, tab in enumerate(tabs):
                    pad[lvl, :nc] = tab.cpu().numpy()
                self._deq_host.append(pad)
        self.occupancy = occupancy.to(torch.uint8).contiguous()
        n0 = self._resolutions[0][::-1]
        want = tuple(-(-(n - 1) // self.block) for n in n0)
        if tuple(self.occupancy.shape) != want:
            raise ValueError(f"occupancy {tuple(self.occupancy.shape)}: need {want} for block {self.block}")
        self.kept_density: Optional[List[torch.Tensor]] = None  # trainable: per level [M_l] in row order
        self._kept_pos: List[torch.Tensor] = []
        self._synced: List[int] = []

    # ---- fine-tuning: the kept points' densities and SH rows as parameters -----------------------------------------

    def requires_grad_(self, requires_grad: bool = True) -> "BakedGrid":
        """Make the grid trainable: per level a contiguous fp32 leaf `kept_density[l]` [M_l] (the kept points'
        densities in SH-row order) and `sh[l]` requiring grad.  The cells follow `kept_density` on the next read
        (`_struct`, `density`, `save`): projected onto >= 0, scattered into the kept points, occupancy rebuilt.  The
        kept set and the rows never change.  False syncs and turns the parameters back into plain tensors.  A quantized
        grid is not trainable: fine-tune before `quantize`, or train `dequantize()`."""
        if requires_grad:
            self._refuse_sparse("requires_grad_")
        if requires_grad and self.quantized:
            raise ValueError("BakedGrid.requires_grad_: a quantized grid is not trainable; the order is bake -> prune -> "
                             "fine-tune -> quantize, or fine-tune dequantize()")
        if not requires_grad:
            if self.kept_density is not None:
                self._sync()
                self.kept_density, self._kept_pos, self._synced = None, [], []
            for c in self.sh:
                c.requires_grad_(False)
            return self
        if self.kept_density is not None:
            return self
        kd, pos = [], self._row_positions()
        for lvl, p in enumerate(pos):
            kd.append(self.cells[lvl].view(-1, 2)[p, 0].view(torch.float32).requires_grad_(True))
            self.sh[lvl].requires_grad_(True)
        self.kept_density, self._kept_pos = kd, pos
        self._synced = [t._version for t in kd]
        return self

    def _row_positions(self) -> List[torch.Tensor]:
        """Per level the int64 lattice position (x fastest) of each SH row, [M_l] in row order; a trainable grid's are
        built once, in `requires_grad_`."""
        if self.kept_density is not None:
            return self._kept_pos
        pos = []
        for lvl in range(self.levels):
            idx = self.cells[lvl][..., 1].reshape(-1)
            flat = (idx >= 0).nonzero().reshape(-1)
            p = torch.empty_like(flat)
            p[idx[flat].long()] = flat  # the lattice position of row r
            pos.append(p)
        return pos

    def total_variation(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(TV_density, TV_sh) as 0-dim fp32 tensors: the total-variation prior of Plenoxels on each level's own
        lattice, on mipnerf_b200_grid_tv.  For each kept point p and axis a, with q = p + e_a its forward neighbour,
        D_a = sigma(q) - sigma(p) (a dropped q reads 0, the density the renderer interpolates there) and D_a c_{k,ch} =
        c_{k,ch}(q) - c_{k,ch}(p) (0 where q is dropped: a dropped point has no row); both are 0 where q lies outside
        the lattice.  TV_density = (1/M) sum_l sum_p sqrt(TV_EPS + sum_a D_a^2) and TV_sh = (1/M) sum_l sum_p
        sum_{k,ch} sqrt(TV_EPS + sum_a (D_a c_{k,ch})^2), M the kept points of all levels (both 0 when M = 0).  On a
        trainable grid in grad mode both are differentiable in `parameters()`; the gradient is bit-reproducible.  A
        trainable grid is synced first.  Not on a sparse or quantized grid: fine-tune before `quantize` and
        `sparsify`."""
        self._refuse_sparse("total_variation")
        self._refuse_quantized("total_variation")
        if self.kept_density is None or not torch.is_grad_enabled():
            with torch.no_grad():
                return _tv_terms(self, self._row_positions())
        self._sync()
        return _GridTV.apply(self, *self.parameters())

    @property
    def trainable(self) -> bool:
        return self.kept_density is not None

    @property
    def quantized(self) -> bool:
        """Whether the SH rows are uint8 (`quantize`)."""
        return self.sh_scale is not None

    @property
    def sparse(self) -> bool:
        """Whether the cells are 8^3-point bricks (`sparsify`)."""
        return self.bricks is not None

    def parameters(self) -> List[torch.Tensor]:
        """[kept_density_0, sh_0, kept_density_1, sh_1, ...] of a trainable grid."""
        if self.kept_density is None:
            raise RuntimeError("BakedGrid.parameters: call requires_grad_() first")
        return [t for pair in zip(self.kept_density, self.sh) for t in pair]

    @torch.no_grad()
    def _sync(self) -> None:
        """Bring the cells and occupancy up to `kept_density` if it changed since the last sync."""
        if self.kept_density is None or [t._version for t in self.kept_density] == self._synced:
            return
        for lvl, (kd, p) in enumerate(zip(self.kept_density, self._kept_pos)):
            kd.clamp_(min=0)
            self.cells[lvl].view(-1, 2)[p, 0] = kd.view(torch.int32)
        self.occupancy = grid_occupancy([self.cells[lvl][..., 0].view(torch.float32) for lvl in range(self.levels)],
                                        self.block)
        self._synced = [t._version for t in self.kept_density]

    @property
    def levels(self) -> int:
        return len(self.sh)

    @property
    def device(self) -> torch.device:
        return self.sh[0].device

    @property
    def resolutions(self) -> List[Tuple[int, int, int]]:
        """(nx, ny, nz) per level."""
        return list(self._resolutions)

    def density(self, level: int = 0) -> torch.Tensor:
        """The baked density [nz, ny, nx] of a level: a view of a dense grid's cells, or on a sparse grid a copy
        rebuilt from the bricks."""
        if self.sparse:
            return self._dense_cells(level)[..., 0].view(torch.float32)
        self._sync()
        return self.cells[level][..., 0].view(torch.float32)

    def index(self, level: int = 0) -> torch.Tensor:
        """The SH row of each lattice point [nz, ny, nx] int32, -1 where not kept: a view of a dense grid's cells, or
        on a sparse grid a copy rebuilt from the bricks."""
        if self.sparse:
            return self._dense_cells(level)[..., 1]
        return self.cells[level][..., 1]

    def _dense_cells(self, level: int, slab_bytes: int = _SLAB_BYTES) -> torch.Tensor:
        """Level `level`'s [nz, ny, nx, 2] cells rebuilt from a sparse grid's bricks, in slabs of brick layers."""
        table, pool = self.bricks[level]
        nz, ny, nx = self._resolutions[level][::-1]
        cells = torch.empty(nz, ny, nx, 2, dtype=torch.int32, device=table.device)
        for z0, slab in _cell_slabs(table, pool, self._resolutions[level], _slab_layers(*table.shape[1:], slab_bytes)):
            cells[z0:z0 + slab.shape[0]] = slab
        return cells

    @property
    def kept(self) -> List[int]:
        return [int(s.shape[0]) for s in self.sh]

    @property
    def nbytes(self) -> int:
        """Bytes held: cells (dense array, or brick pools and tables), SH rows, quantization tables and occupancy."""
        tables = self.sh_scale + self.sh_offset if self.quantized else []
        cells = [t for pair in self.bricks for t in pair] if self.sparse else self.cells
        return sum(t.numel() * t.element_size() for t in cells + self.sh + tables) + self.occupancy.numel()

    def default_step(self) -> float:
        """Half the finest level's smallest voxel edge."""
        _, step = lattice_axes(self.resolutions[0], self.bounds, "cpu")
        return float(np.float32(0.5) * step.min())

    def _struct(self) -> "_cabi.Grid":
        self._sync()
        g = _cabi.Grid()
        for lvl, (s, (nx, ny, nz)) in enumerate(zip(self.sh, self._resolutions)):
            fp32_rows = s.data_ptr() if s.numel() and not self.quantized else None  # a quantized grid's are in _sh_u8
            cells = None if self.sparse else self.cells[lvl].data_ptr()  # a sparse grid's are in _bricks
            g.levels[lvl] = _cabi.GridLevel(cells, fp32_rows, nx, ny, nz)
        g.num_levels, g.degree = self.levels, self.degree
        g.lo = (C.c_float * 3)(*self.bounds[0])
        g.hi = (C.c_float * 3)(*self.bounds[1])
        g.rgb_padding, g.occupancy, g.block = self.rgb_padding, self.occupancy.data_ptr(), self.block
        return g

    def _sh_u8(self) -> "_cabi.GridShU8":
        """The uint8 rows and the scale / offset values of a quantized grid, as mipnerf_b200_grid_render_u8 takes them."""
        t = _cabi.GridShU8()
        for lvl, s in enumerate(self.sh):
            t.rows[lvl] = s.data_ptr() if s.numel() else None
        scale, offset = self._deq_host
        C.memmove(C.addressof(t.scale), scale.ctypes.data, scale.nbytes)
        C.memmove(C.addressof(t.offset), offset.ctypes.data, offset.nbytes)
        return t

    def _bricks_struct(self) -> "_cabi.GridBricks":
        """The brick tables and pools of a sparse grid, as mipnerf_b200_grid_render_bricks takes them."""
        b = _cabi.GridBricks()
        for lvl, (table, pool) in enumerate(self.bricks):
            b.table[lvl] = table.data_ptr()
            b.pool[lvl] = pool.data_ptr() if pool.numel() else None
        return b

    def render(self, rays: Rays, white_bkgd: bool = True, step: Optional[float] = None):
        """(rgb [B,3], distance [B], acc [B]) of flat rays on the grid's device, marched every `step` along |d| (default
        `default_step()`).  Differentiable in `parameters()` when the grid is trainable and grad mode is on (rays that
        require grad are refused: there is no ray gradient).  A quantized grid renders on
        mipnerf_b200_grid_render_u8, bit for bit as its `dequantize()` renders; a sparse grid on
        mipnerf_b200_grid_render_bricks, bit for bit as its `densify()` renders."""
        if self.kept_density is None or not torch.is_grad_enabled():
            with torch.no_grad():
                return self._render(rays, white_bkgd, step)[0]
        if any(isinstance(f, torch.Tensor) and f.requires_grad for f in rays):
            raise ValueError("BakedGrid.render: rays that require grad; the grid has no gradient for rays")
        self._sync()
        return _GridRender.apply(self, rays, bool(white_bkgd), step, *self.parameters())

    def _render(self, rays: Rays, white_bkgd: bool, step: Optional[float]):
        """((rgb, distance, acc), the fp32 ray fields the launch read, the step it used)."""
        dev = _dev(self.sh[0])
        rs, keep = _grid_rays(rays, dev)
        n = rs.num_rays
        g = self._struct()
        rgb = torch.empty(n, 3, device=dev)
        dist = torch.empty(n, device=dev)
        acc = torch.empty(n, device=dev)
        st = self.default_step() if step is None else float(step)
        out = (int(bool(white_bkgd)), rgb.data_ptr(), dist.data_ptr(), acc.data_ptr())
        if self.sparse:
            _call(dev, "grid_render_bricks", _cabi.lib().mipnerf_b200_grid_render_bricks, C.byref(g),
                  C.byref(self._bricks_struct()), C.byref(self._sh_u8()) if self.quantized else None, C.byref(rs), st,
                  *out)
        elif self.quantized:
            _call(dev, "grid_render_u8", _cabi.lib().mipnerf_b200_grid_render_u8, C.byref(g), C.byref(self._sh_u8()),
                  C.byref(rs), st, *out)
        else:
            _call(dev, "grid_render", _cabi.lib().mipnerf_b200_grid_render, C.byref(g), C.byref(rs), st, *out)
        return (rgb, dist, acc), keep, st

    def visibility(self, rays: Rays, step: Optional[float] = None,
                   out: Optional[Sequence[torch.Tensor]] = None) -> List[torch.Tensor]:
        """Per level an fp32 [M_l] tensor (SH-row order) of each kept point's largest score over `rays`: at every
        composited sample of `render`'s march, blending weight T_k alpha_k times the coefficient the renderer gives the
        point's colour (level weight times trilinear weight).  With `out` (such tensors, e.g. from an earlier call),
        the scores are raised into it in place and it is returned, so calls over batches of rays accumulate.  The
        result is bit-reproducible under any order or split of the rays.  `step` defaults to `default_step()` as in
        `render`; a prune by these scores only holds for renders at the same step.  Not on a quantized or sparse grid:
        prune before `quantize` and `sparsify`."""
        self._refuse_sparse("visibility")
        self._refuse_quantized("visibility")
        dev = _dev(self.cells[0])
        if out is None:
            out = [torch.zeros(m, device=dev) for m in self.kept]
        else:
            out = list(out)
            if len(out) != self.levels or any(
                    t.dtype != torch.float32 or t.device != dev or tuple(t.shape) != (m,) or not t.is_contiguous()
                    for t, m in zip(out, self.kept)):
                raise ValueError(f"out: need {self.levels} contiguous fp32 tensors of shapes {self.kept} on {dev}")
        self._visibility(rays, step, out)
        return out

    def _visibility(self, rays: Rays, step: Optional[float], out: Sequence[torch.Tensor]) -> None:
        """`visibility`'s launch into `out`, on dense cells or (mipnerf_b200_grid_visibility_bricks) bricks.  It reads
        no SH row, so `out` may be sized for rows not baked yet."""
        dev = _dev(self.sh[0])
        rs, keep = _grid_rays(rays, dev)
        g, mw = self._struct(), _level_ptrs(out)
        st = self.default_step() if step is None else float(step)
        if self.sparse:
            _call(dev, "grid_visibility_bricks", _cabi.lib().mipnerf_b200_grid_visibility_bricks, C.byref(g),
                  C.byref(self._bricks_struct()), C.byref(rs), st, mw)
        else:
            _call(dev, "grid_visibility", _cabi.lib().mipnerf_b200_grid_visibility, C.byref(g), C.byref(rs), st, mw)

    def proposal(self, rays: Rays, t_samples: torch.Tensor, differentiable: bool = False) -> torch.Tensor:
        """Proposal weights [B, N] of flat `rays` at fenceposts `t_samples` [B, N+1] (1 <= N <= 256), on
        mipnerf_b200_grid_proposal: per interval, the grid's density at its midpoint under the renderer's level blend,
        composited as volumetric_rendering's weights with no early stop.  What `MipNerf.forward_proposed` resamples
        level 1 from.  Dense, sparse, quantized and trainable grids (synced first); no gradient.  With
        `differentiable`, on a trainable grid in grad mode, the weights carry a graph in `kept_density`
        (mipnerf_b200_grid_proposal_backward, what `finetune_proposal` trains through): the SH rows get no gradient,
        and rays or fenceposts that require grad are refused, as they have none.  Anywhere else `differentiable`
        changes nothing."""
        if not differentiable or self.kept_density is None or not torch.is_grad_enabled():
            with torch.no_grad():
                return self._proposal(rays, t_samples)[0]
        if t_samples.requires_grad or any(isinstance(f, torch.Tensor) and f.requires_grad for f in rays):
            raise ValueError("BakedGrid.proposal: rays or t_samples that require grad; the grid has no gradient for "
                             "them")
        self._sync()
        return _GridProposal.apply(self, rays, t_samples, *self.parameters())

    def _proposal(self, rays: Rays, t_samples: torch.Tensor):
        """(weights, the fp32 ray fields the launch read, the fp32 fenceposts it read)."""
        dev = _dev(self.sh[0])
        rs, keep = _grid_rays(rays, dev)
        b = rs.num_rays
        if t_samples.dim() != 2 or t_samples.shape[0] != b or not 2 <= t_samples.shape[1] <= 257:
            raise ValueError(f"t_samples {tuple(t_samples.shape)}: need [B = {b}, N + 1] with 1 <= N <= 256")
        if t_samples.device != dev:
            raise ValueError(f"t_samples on {t_samples.device}, grid on {dev}")
        t = _f32(t_samples)
        n = t.shape[1] - 1
        out = torch.empty(b, n, device=dev)
        _call(dev, "grid_proposal", _cabi.lib().mipnerf_b200_grid_proposal, C.byref(self._struct()),
              C.byref(self._bricks_struct()) if self.sparse else None, C.byref(rs), t.data_ptr(), n, out.data_ptr())
        return out, keep, t

    @torch.no_grad()
    def prune(self, max_weight: Sequence[torch.Tensor], weight_threshold: float) -> "BakedGrid":
        """A new, non-trainable grid that keeps the points kept here whose score in `max_weight` (per level [M_l] in
        SH-row order, as `visibility` returns) is > `weight_threshold`; `self` is left as it is.  A point pruned away
        gets density 0 and index -1; the kept points' rows are renumbered in x-fastest order and their SH rows carried
        over bit for bit; the occupancy is rebuilt by `grid_occupancy`; bounds, degree, rgb_padding and block are
        copied.  Plain torch on the grid's device (CPU tensors too).  Not on a quantized or sparse grid: prune before
        `quantize` and `sparsify`."""
        self._refuse_sparse("prune")
        self._refuse_quantized("prune")
        self._sync()
        if len(max_weight) != self.levels:
            raise ValueError(f"max_weight: {len(max_weight)} levels, the grid has {self.levels}")
        dens, indices, sh = [], [], []
        for lvl, (mw, m) in enumerate(zip(max_weight, self.kept)):
            if tuple(mw.shape) != (m,):
                raise ValueError(f"max_weight[{lvl}]: shape {tuple(mw.shape)}, need ({m},)")
            old = self.index(lvl)
            d = self.density(lvl)
            kept = old >= 0
            keep = kept.clone()
            keep[kept] = mw.to(d.device)[old[kept].long()] > float(weight_threshold)
            idx = torch.full_like(old, -1)
            idx[keep] = torch.arange(int(keep.sum()), dtype=old.dtype, device=old.device)
            dens.append(torch.where(kept & ~keep, torch.zeros((), device=d.device), d))
            indices.append(idx)
            sh.append(self.sh[lvl].detach()[old[keep].long()])  # x-fastest order of the kept points
        return self._derive(dense=(dens, indices), sh=sh, occupancy=grid_occupancy(dens, self.block))

    def _refuse_sparse(self, what: str) -> None:
        if self.sparse:
            raise ValueError(f"BakedGrid.{what}: the grid is sparse (brick cells); the order is bake -> prune -> "
                             f"fine-tune -> quantize -> sparsify, or use densify()")

    def _refuse_quantized(self, what: str) -> None:
        if self.quantized:
            raise ValueError(f"BakedGrid.{what}: the grid is quantized; the order is bake -> prune -> fine-tune -> "
                             f"quantize, or use dequantize()")

    @torch.no_grad()
    def quantize(self) -> "BakedGrid":
        """A new, non-trainable grid whose SH rows are uint8, with per level, coefficient and channel offset = the
        column's minimum over the kept rows and scale = (max - min) / 255 (fp32), and q = clamp(round((c - offset) /
        scale), 0, 255), 0 where scale == 0; a level without kept rows gets scale = offset = 0.  Each coefficient then
        reads as fl(fl(q * scale) + offset), within scale / 2 (plus a few ulp of the column's magnitude) of c.  A
        trainable grid is synced first and its detached values are used; `self` is left as it is.  The cells,
        indices, occupancy, bounds, degree, rgb_padding and block are copied.  Plain, deterministic torch on the
        grid's device (CPU tensors too).  Non-finite rows are refused.  Not on a sparse grid."""
        self._refuse_sparse("quantize")
        if self.quantized:
            raise ValueError("BakedGrid.quantize: the grid is already quantized")
        self._sync()
        rows, scales, offsets = zip(*[_quantize_rows(c.detach(), lvl) for lvl, c in enumerate(self.sh)])
        return self._derive(sh=rows, sh_tables=(scales, offsets))

    @torch.no_grad()
    def dequantize(self) -> "BakedGrid":
        """The fp32 grid of a quantized one: SH rows fl(fl(q * scale) + offset) (eager torch: one rounded multiply,
        then one rounded add), everything else copied.  It renders bit for bit as the quantized grid does.  Not on a
        sparse grid."""
        self._refuse_sparse("dequantize")
        if not self.quantized:
            raise ValueError("BakedGrid.dequantize: the grid is not quantized (fp32 rows)")
        rows = [q.to(torch.float32) * s + o for q, s, o in zip(self.sh, self.sh_scale, self.sh_offset)]
        return self._derive(sh=rows, sh_tables=(None, None))

    @torch.no_grad()
    def sparsify(self, slab_bytes: int = _SLAB_BYTES) -> "BakedGrid":
        """A new grid whose cells keep only each level's non-empty bricks of 8^3 lattice points (module docstring,
        "Memory layout"); `self` is left as it is.  Lossless: it renders bit for bit as `self`, and `densify()` gives
        back every array bit for bit.  The SH rows (fp32 or uint8), quantization tables, occupancy, bounds, degree,
        rgb_padding and block are copied.  A trainable grid is synced first and its detached values are used.  Plain,
        deterministic torch on the grid's device (CPU tensors too), in slabs of brick layers of about `slab_bytes`
        bytes of dense cells each, so that its transient memory stays near the size of the result."""
        if self.sparse:
            raise ValueError("BakedGrid.sparsify: the grid is already sparse")
        self._sync()
        tables, pools = [], []
        for c in self.cells:
            nz, ny, nx = c.shape[:3]
            t = (-(-nz // BRICK), -(-ny // BRICK), -(-nx // BRICK))
            step = _slab_layers(t[1], t[2], slab_bytes)
            table = torch.empty(t, dtype=torch.int32, device=c.device)
            count = 0
            for z0 in range(0, t[0], step):  # the table: stored bricks numbered in raster order
                z1 = min(z0 + step, t[0])
                table[z0:z1], _, count = _number_bricks(_brick_slab(c, z0, z1, t), count)
            pool = torch.empty(count, BRICK, BRICK, BRICK, 2, dtype=torch.int32, device=c.device)
            for z0 in range(0, t[0], step):  # the pool, filled slab by slab
                z1 = min(z0 + step, t[0])
                tab = table[z0:z1]
                stored = tab >= 0
                pool[tab[stored].long()] = _brick_slab(c, z0, z1, t)[stored]
            tables.append(table)
            pools.append(pool)
        return self._derive(bricks=(tables, pools))

    @torch.no_grad()
    def densify(self, slab_bytes: int = _SLAB_BYTES) -> "BakedGrid":
        """The dense grid of a sparse one (`sparsify`'s inverse, bit for bit in every array), in slabs of brick
        layers; `self` is left as it is."""
        if not self.sparse:
            raise ValueError("BakedGrid.densify: the grid is not sparse (dense cells)")
        cells = [self._dense_cells(lvl, slab_bytes) for lvl in range(self.levels)]
        return self._derive(dense=([c[..., 0].view(torch.float32) for c in cells], [c[..., 1] for c in cells]))

    def _derive(self, dense=None, bricks=None, sh=None, sh_tables=None, occupancy=None) -> "BakedGrid":
        """A new grid with this grid's bounds, degree, rgb_padding and block, and a copy of each other part not given:
        cells (`dense` = (densities, indices) or `bricks` = (tables, pools), per level), SH rows, quantization tables
        (`sh_tables` = (sh_scale, sh_offset), (None, None) for fp32 rows) and occupancy."""
        if dense is None and bricks is None:
            dense = ([self.density(lvl) for lvl in range(self.levels)], [self.index(lvl) for lvl in range(self.levels)])
        if sh_tables is None:
            q = self.quantized
            sh_tables = ([s.clone() for s in self.sh_scale], [o.clone() for o in self.sh_offset]) if q else (None, None)
        shared = ([s.detach().clone() for s in self.sh] if sh is None else sh,
                  self.occupancy.clone() if occupancy is None else occupancy, self.bounds, self.degree,
                  self.rgb_padding, self.block, *sh_tables)
        if bricks is not None:
            return BakedGrid.from_bricks(*bricks, self.resolutions, *shared)
        return BakedGrid(*dense, *shared)

    def save(self, path: str) -> None:
        """One .npz: per level density, index and sh, plus occupancy, bounds, degree, rgb_padding and block (format
        1).  A quantized grid writes format 2: sh_{l} is its uint8 rows, plus sh_scale_{l} and sh_offset_{l} fp32
        [(degree + 1)^2, 3].  A sparse grid writes format 3: per level table_{l} and pool_{l} in place of density_{l}
        and index_{l}, `resolutions` int32 [levels, 3] (nx, ny, nz), and its rows as format 1 or 2 does."""
        self._sync()
        fmt = _FORMAT_BRICKS if self.sparse else _FORMAT_U8 if self.quantized else _FORMAT
        arrays = {"format": np.int32(fmt), "levels": np.int32(self.levels), "degree": np.int32(self.degree),
                  "rgb_padding": np.float32(self.rgb_padding), "block": np.int32(self.block),
                  "bounds": np.asarray(self.bounds, dtype=np.float32), "occupancy": self.occupancy.cpu().numpy()}
        if self.sparse:
            arrays["resolutions"] = np.asarray(self._resolutions, dtype=np.int32)
        for lvl in range(self.levels):
            if self.sparse:
                arrays[f"table_{lvl}"] = self.bricks[lvl][0].cpu().numpy()
                arrays[f"pool_{lvl}"] = self.bricks[lvl][1].cpu().numpy()
            else:
                arrays[f"density_{lvl}"] = self.density(lvl).cpu().numpy()
                arrays[f"index_{lvl}"] = self.index(lvl).cpu().numpy()
            arrays[f"sh_{lvl}"] = self.sh[lvl].detach().cpu().numpy()
            if self.quantized:
                arrays[f"sh_scale_{lvl}"] = self.sh_scale[lvl].cpu().numpy()
                arrays[f"sh_offset_{lvl}"] = self.sh_offset[lvl].cpu().numpy()
        np.savez(path, **arrays)

    @classmethod
    def load(cls, path: str, device="cuda") -> "BakedGrid":
        with np.load(path) as z:
            fmt = int(z["format"])
            if fmt not in (_FORMAT, _FORMAT_U8, _FORMAT_BRICKS):
                raise ValueError(f"{path}: baked-grid format {fmt}, this library reads {_FORMAT}, {_FORMAT_U8} and "
                                 f"{_FORMAT_BRICKS}")
            levels = int(z["levels"])
            t = lambda name: torch.from_numpy(np.ascontiguousarray(z[name])).to(device)  # noqa: E731
            bounds = z["bounds"].astype(np.float64)
            tables = {}
            if fmt == _FORMAT_U8 or fmt == _FORMAT_BRICKS and "sh_scale_0" in z.files:
                tables = {"sh_scale": [t(f"sh_scale_{lvl}") for lvl in range(levels)],
                          "sh_offset": [t(f"sh_offset_{lvl}") for lvl in range(levels)]}
            if fmt == _FORMAT_BRICKS:
                want = ["resolutions"] + [f"{k}_{lvl}" for lvl in range(levels) for k in ("table", "pool", "sh")]
                missing = [k for k in want if k not in z.files]
                if missing:
                    raise ValueError(f"{path}: baked-grid format {fmt} without its arrays {missing}")
                return cls.from_bricks([t(f"table_{lvl}") for lvl in range(levels)],
                                       [t(f"pool_{lvl}") for lvl in range(levels)],
                                       [tuple(int(n) for n in r) for r in z["resolutions"]],
                                       [t(f"sh_{lvl}") for lvl in range(levels)], t("occupancy"),
                                       (tuple(bounds[0]), tuple(bounds[1])), int(z["degree"]), float(z["rgb_padding"]),
                                       int(z["block"]), **tables)
            return cls([t(f"density_{lvl}") for lvl in range(levels)], [t(f"index_{lvl}") for lvl in range(levels)],
                       [t(f"sh_{lvl}") for lvl in range(levels)], t("occupancy"),
                       (tuple(bounds[0]), tuple(bounds[1])), int(z["degree"]), float(z["rgb_padding"]), int(z["block"]),
                       **tables)


@torch.no_grad()
def _quantize_rows(c: torch.Tensor, lvl: int, chunk_rows: int = 1 << 16):
    """The 8-bit codec of one level's fp32 SH rows [M, nc, 3] (`BakedGrid.quantize`) -> (uint8 rows [M, nc, 3],
    scale [nc, 3], offset [nc, 3]).  The checks, column extremes and codes run `chunk_rows` rows at a time (a minimum
    or maximum of chunk extremes is the column's, exactly), so that the transient memory is a few fp32 chunks rather
    than copies of the rows."""
    nc = c.shape[1]
    chunks = [c[s:s + chunk_rows] for s in range(0, c.shape[0], chunk_rows)]
    if not all(bool(torch.isfinite(x).all()) for x in chunks):
        raise ValueError(f"BakedGrid.quantize: level {lvl} has non-finite SH coefficients")
    if c.shape[0] == 0:
        scale = offset = torch.zeros(nc, 3, device=c.device)
        return torch.empty(0, nc, 3, dtype=torch.uint8, device=c.device), scale, offset
    offset = torch.stack([x.amin(dim=0) for x in chunks]).amin(dim=0)
    hi = torch.stack([x.amax(dim=0) for x in chunks]).amax(dim=0)
    # a tensor divisor: CUDA torch turns a Python-scalar divisor into a multiply by its reciprocal, which is not the
    # correctly rounded quotient the CPU gives
    scale = (hi - offset) / torch.full_like(hi, 255.0)
    if not bool(torch.isfinite(scale).all()):
        raise ValueError(f"BakedGrid.quantize: level {lvl}: a column's range overflows fp32")
    live = scale > 0
    div = torch.where(live, scale, torch.ones((), device=c.device))
    q = torch.empty(c.shape, dtype=torch.uint8, device=c.device)
    for s in range(0, c.shape[0], chunk_rows):
        code = torch.round((c[s:s + chunk_rows] - offset) / div)
        q[s:s + chunk_rows] = torch.where(live, code.clamp(0, 255), torch.zeros((), device=c.device)).to(torch.uint8)
    return q, scale, offset


def _slab_layers(ty: int, tx: int, slab_bytes: int) -> int:
    """Brick layers per slab: as many as fit `slab_bytes` of dense cells, at least one."""
    return max(1, int(slab_bytes) // (ty * tx * BRICK ** 3 * 8))


def _empty_words(shape, device) -> torch.Tensor:
    """[*shape, 2] int32 whose every word is (+0.0 bits, -1), the word of a point that is not kept."""
    w = torch.empty(*shape, 2, dtype=torch.int32, device=device)
    w[..., 0] = 0
    w[..., 1] = -1
    return w


def _brick_slab(cells: torch.Tensor, z0: int, z1: int, t) -> torch.Tensor:
    """Brick layers [z0, z1) of dense cells [nz, ny, nx, 2] as [z1 - z0, ty, tx, 8, 8, 8, 2] (a view of a padded
    copy), points past the lattice holding (0, -1)."""
    nz, ny, nx = cells.shape[:3]
    pad = _empty_words(((z1 - z0) * BRICK, t[1] * BRICK, t[2] * BRICK), cells.device)
    zs = cells[z0 * BRICK:min(z1 * BRICK, nz)]
    pad[:zs.shape[0], :ny, :nx] = zs
    return pad.view(z1 - z0, BRICK, t[1], BRICK, t[2], BRICK, 2).permute(0, 2, 4, 1, 3, 5, 6)


def _cell_slabs(table: torch.Tensor, pool: torch.Tensor, resolution, step: int):
    """A level's dense cells rebuilt from its bricks (table [tz, ty, tx], pool [num_bricks, 8, 8, 8, 2], `resolution`
    (nx, ny, nz)), `step` brick layers at a time: yields (z0, cells [zn, ny, nx, 2] of lattice layers [z0, z0 + zn))."""
    nz, ny, nx = resolution[::-1]
    tz, ty, tx = table.shape
    for b0 in range(0, tz, step):
        b1 = min(b0 + step, tz)
        tab = table[b0:b1]
        b = _empty_words((b1 - b0, ty, tx, BRICK, BRICK, BRICK), table.device)
        stored = tab >= 0
        b[stored] = pool[tab[stored].long()]
        dense = b.permute(0, 3, 1, 4, 2, 5, 6).reshape((b1 - b0) * BRICK, ty * BRICK, tx * BRICK, 2)
        zn = min(b1 * BRICK, nz) - b0 * BRICK
        yield b0 * BRICK, dense[:zn, :ny, :nx]


_PRUNE_CHUNK = 1 << 10  # _prune_bricks: bricks rewritten at once


@torch.no_grad()
def _prune_bricks(tables, pools, positions, resolutions, scores, weight_threshold: float, block: int,
                  slab: Optional[int] = None):
    """`BakedGrid.prune(scores, weight_threshold).sparsify()` on the structure `sparse_grid_structure` returns (per
    level the brick table, pool and kept positions, and the scores [M_l] of the kept points in SH-row order) ->
    (tables, pools, positions, occupancy), every array bit for bit as that path gives it.  A kept point survives iff
    its score is > weight_threshold, and the survivors are renumbered in row order (x fastest already).  A dropped
    point's word becomes (+0.0 bits, -1), a brick left with only such words is dropped, and the stored bricks stay in
    raster order.  The occupancy is rebuilt from the pruned bricks in slabs of `slab` brick layers (None: the whole
    level).  The lists `pools`, `positions` and `scores` are consumed: each pool is rewritten in place, and each level's
    entries are released once its pruned arrays exist, so that a level's pool is held twice only while it is
    compacted."""
    o = tuple(-(-(n - 1) // int(block)) for n in resolutions[0][::-1])
    out_tables, out_pools, out_positions = [], [], []
    for lvl, table in enumerate(tables):
        pool = pools[lvl]
        keep = scores[lvl] > float(weight_threshold)
        scores[lvl] = None
        rowmap = torch.cumsum(keep, 0, dtype=torch.int32) - 1  # the new row of a surviving old row
        rowmap[~keep] = -1
        out_positions.append(positions[lvl][keep])
        positions[lvl] = None
        del keep
        ids, count = [], 0
        for s in range(0, pool.shape[0], _PRUNE_CHUNK):
            w = pool[s:s + _PRUNE_CHUNK]
            row = w[..., 1]
            live = row >= 0
            new = torch.full_like(row, -1)
            new[live] = rowmap[row[live].long()]
            w[..., 0].masked_fill_(live & (new < 0), 0)
            w[..., 1] = new
            tab, _, count = _number_bricks(w[None, None], count)
            ids.append(tab.reshape(-1))
        del rowmap
        if pool.shape[0]:
            ids = torch.cat(ids)  # the new id of each old brick, -1 for a brick left empty
            out_pools.append(pool[ids >= 0])
            out_tables.append(torch.where(table >= 0, ids[table.clamp(min=0).long()], table))
        else:
            out_pools.append(pool)
            out_tables.append(table.clone())
        pools[lvl] = pool = None
    occ = torch.zeros(o, dtype=torch.bool, device=tables[0].device)
    for lvl, (table, pool, r) in enumerate(zip(out_tables, out_pools, resolutions)):
        for z0, cells in _cell_slabs(table, pool, r, table.shape[0] if slab is None else int(slab)):
            occ |= _occupancy_counts((cells[..., 0].view(torch.float32) != 0).to(torch.float32), z0, r[2], o,
                                     int(block), 1 << lvl) > 0
    return out_tables, out_pools, out_positions, occ.to(torch.uint8)


def _number_bricks(bricks: torch.Tensor, count: int):
    """The table entries of a slab of bricks [z, ty, tx, 8, 8, 8, 2] (`_brick_slab`) whose stored bricks are numbered
    from `count` in raster order -> (int32 table slab [z, ty, tx], stored mask, count after the slab).  A brick is
    stored iff one of its words is not (+0.0 bits, -1)."""
    stored = ((bricks[..., 0] != 0) | (bricks[..., 1] != -1)).flatten(3).any(-1)
    ids = torch.cumsum(stored.reshape(-1), 0).view(stored.shape) - 1 + count
    table = torch.where(stored, ids, torch.full((), -1, device=bricks.device)).to(torch.int32)
    return table, stored, count + int(stored.sum())


def _grid_rays(rays: Rays, dev: torch.device):
    """(RaysStruct, keep) of flat `rays` (`_rays_struct`) for a launch on the grid's device `dev`."""
    o = rays.origins.reshape(-1, 3)
    if o.device != dev:
        raise ValueError(f"rays on {o.device}, grid on {dev}")
    return _rays_struct(o, rays.directions.reshape(-1, 3), rays.viewdirs.reshape(-1, 3), rays.radii.reshape(-1),
                        rays.near.reshape(-1), rays.far.reshape(-1))


def _level_ptrs(ts: Sequence[torch.Tensor]):
    """The per-level pointer array of tensors `ts`, NULL for an empty one."""
    return (C.c_void_p * len(ts))(*[t.data_ptr() if t.numel() else None for t in ts])


def _grid_grads(grads: Sequence[Optional[torch.Tensor]]) -> "_cabi.GridGrads":
    """The GridGrads of gradients in `parameters()` order, NULL for a level without kept points.  An SH gradient of
    None leaves that level's `sh` NULL: density-only gradients."""
    gg = _cabi.GridGrads()
    for lvl in range(len(grads) // 2):
        density, sh = grads[2 * lvl], grads[2 * lvl + 1]
        if density.numel():
            gg.density[lvl] = density.data_ptr()
            if sh is not None:
                gg.sh[lvl] = sh.data_ptr()
    return gg


class _GridRender(torch.autograd.Function):
    """BakedGrid.render of a trainable grid: the forward is the no-grad launch; the backward zeroes one gradient per
    parameter and adds mipnerf_b200_grid_render_backward into them."""

    @staticmethod
    def forward(ctx, grid, rays, white_bkgd, step, *params):
        ctx.set_materialize_grads(False)  # an unused output's cotangent stays None: NULL to the kernel
        out, rays_keep, ctx.step = grid._render(rays, white_bkgd, step)
        ctx.grid, ctx.white_bkgd, ctx.num_rays = grid, white_bkgd, out[0].shape[0]
        # the parameters and the ray fields the kernel reads (aliases of the caller's rays when those are contiguous
        # fp32): an in-place update of either before the backward raises autograd's version error
        ctx.save_for_backward(*params, *rays_keep)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_rgb, d_dist, d_acc):
        saved = ctx.saved_tensors
        params, rays_keep = saved[:-6], saved[-6:]
        grid = ctx.grid
        dev = _dev(grid.cells[0])
        grads = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in params]
        cot = [None if t is None else _f32(t) for t in (d_rgb, d_dist, d_acc)]
        rs = _cabi.RaysStruct(*[t.data_ptr() for t in rays_keep], ctx.num_rays)
        _call(dev, "grid_render_backward", _cabi.lib().mipnerf_b200_grid_render_backward, C.byref(grid._struct()),
              C.byref(rs), ctx.step, int(ctx.white_bkgd), *[None if t is None else t.data_ptr() for t in cot],
              C.byref(_grid_grads(grads)))
        return (None, None, None, None, *grads)


class _GridProposal(torch.autograd.Function):
    """BakedGrid.proposal of a trainable grid: the forward is the no-grad launch; the backward zeroes one gradient per
    kept density and adds mipnerf_b200_grid_proposal_backward into them.  The SH rows get None."""

    @staticmethod
    def forward(ctx, grid, rays, t_samples, *params):
        out, rays_keep, t = grid._proposal(rays, t_samples)
        ctx.grid, ctx.num_rays = grid, out.shape[0]
        # the densities and the ray fields and fenceposts the kernel reads: an in-place update of any of them before the
        # backward raises autograd's version error
        ctx.save_for_backward(*params[0::2], t, *rays_keep)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_weights):
        grid = ctx.grid
        saved = ctx.saved_tensors
        dens, t, rays_keep = saved[:grid.levels], saved[grid.levels], saved[grid.levels + 1:]
        dev = _dev(grid.cells[0])
        grads = [x for d in dens for x in (torch.zeros_like(d, memory_format=torch.contiguous_format), None)]
        gw = _f32(d_weights)
        rs = _cabi.RaysStruct(*[x.data_ptr() for x in rays_keep], ctx.num_rays)
        _call(dev, "grid_proposal_backward", _cabi.lib().mipnerf_b200_grid_proposal_backward, C.byref(grid._struct()),
              C.byref(rs), t.data_ptr(), t.shape[1] - 1, gw.data_ptr(), C.byref(_grid_grads(grads)))
        return (None, None, None, *grads)


def _tv_launch(grid: BakedGrid, pos, terms=None, weights=None, grads=None) -> None:
    """mipnerf_b200_grid_tv on a dense fp32 grid: per-level terms (a pair of lists of [M_l] tensors) and / or the
    weighted gradient (a list [density_0, sh_0, ...] with the shapes of `parameters()`, `weights` a device fp32 [2])."""
    g = grid._struct()
    dev = _dev(grid.cells[0])
    terms = (None, None) if terms is None else [_level_ptrs(t) for t in terms]
    _call(dev, "grid_tv", _cabi.lib().mipnerf_b200_grid_tv, C.byref(g), _level_ptrs(pos),
          (C.c_int64 * grid.levels)(*[p.numel() for p in pos]), TV_EPS, *terms,
          None if weights is None else weights.data_ptr(), None if grads is None else C.byref(_grid_grads(grads)))


def _tv_terms(grid: BakedGrid, pos) -> Tuple[torch.Tensor, torch.Tensor]:
    """(TV_density, TV_sh): the per-point terms summed level by level, in level order, over M."""
    terms = ([torch.empty(p.numel(), device=grid.device) for p in pos],
             [torch.empty(p.numel(), device=grid.device) for p in pos])
    m = sum(p.numel() for p in pos)
    if m == 0:
        return torch.zeros((), device=grid.device), torch.zeros((), device=grid.device)
    _tv_launch(grid, pos, terms=terms)
    return tuple(torch.stack([t.sum() for t in ts]).sum() / m for ts in terms)


class _GridTV(torch.autograd.Function):
    """BakedGrid.total_variation of a trainable grid: the forward launches for the per-point terms and sums them; the
    backward launches once for the gradient of both sums, weighted by the cotangents over M on the device."""

    @staticmethod
    def forward(ctx, grid, *params):
        ctx.grid = grid
        # the parameters the kernel reads: an in-place update before the backward raises autograd's version error
        ctx.save_for_backward(*params)
        return _tv_terms(grid, grid._kept_pos)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_density, d_sh):
        params = ctx.saved_tensors
        grid = ctx.grid
        grads = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in params]
        m = sum(p.numel() for p in grid._kept_pos)
        if m:
            weights = torch.stack([d_density, d_sh]).to(torch.float32) / m
            _tv_launch(grid, grid._kept_pos, weights=weights, grads=grads)
        return (None, *grads)


@torch.no_grad()
def bake_grid(model, resolution: Resolution = 257, levels: int = 1, threshold: float = DEFAULT_THRESHOLD,
              degree: int = 2, n_theta: int = 8, bounds=DEFAULT_BOUNDS, block: int = DEFAULT_BLOCK,
              slab_points: int = 1 << 20, sparse: bool = False, quantize: bool = False,
              stream_points: int = 1 << 24, prune=None,
              weight_threshold: float = DEFAULT_WEIGHT_THRESHOLD) -> BakedGrid:
    """Bake `model` into a `levels`-level grid over `bounds` (level l: (n_0 - 1) / 2^l + 1 points per axis): the
    density of `field.density_grid` at its default voxel variance, the keep mask, index and occupancy of
    `grid_structure`, and the raw SH colour of the kept points' voxel Gaussians (`field.bake_sh(raw=True)`, degree
    0..3, in slabs of `slab_points`), on the model's device.

    `quantize`: the result of `.quantize()` on that grid.  `sparse`: the result of `.sparsify()` on it (after
    `quantize`), bit for bit in every array, but baked without ever holding an array the size of a level's lattice:
    `sparse_grid_structure` walks each level in z-slabs of brick layers, querying `density_grid(z_range=...)` on
    each slab plus one layer of halo, then the kept points' SH rows are baked as above (quantized level by level once
    a level's fp32 rows are all baked).  A slab is L = max(1, stream_points // (512 ty tx)) brick layers, with (tx,
    ty) = ceil((nx, ny) / 8) of level 0 (coarser levels' slabs are smaller).  With P = (8 L + 2) (8 ty) (8 tx) the
    points of level 0's slab padded to bricks with its halo, Q = min(P, max(2^22, nx ny)) the points of one density
    query, M the kept points of all levels, M_l and B_l the kept points and stored bricks of level l, and nc = (degree
    + 1)^2, the memory held at once beyond the returned grid, the model and the queries' workspace is at most

        8 M + max(64 P + 28 Q + max_l (8 M_l + 4096 B_l),
                  (72 + 12 nc) slab_points + [quantize] 12 nc (max_l M_l + 2^19))

    bytes: per slab the densities, masks, cells and padded bricks, the positions of the kept points until their rows
    are baked (8 M), one level's positions and pool twice while their slabs are joined, and one SH query's points and
    output (or with `quantize` one level's fp32 rows and the codec's temporaries of 2^16 rows).  The dense bake holds
    at least 20 bytes per point of level 0's whole lattice at once.

    `prune` (a `DeviceRayBank`, or None): the result of `prune_grid(grid, prune, weight_threshold)` on the unquantized
    dense grid, then `quantize` and `sparse` as above (bake -> prune -> quantize -> sparsify), bit for bit in every
    array; the visibility runs at `default_step()`.  The visibility and the prune run on the structure, before any SH
    row is baked, so only the surviving points' rows are queried.  With `sparse` the visibility reads the bricks
    (mipnerf_b200_grid_visibility_bricks) and no array the size of a level's lattice is held either.  With M' and B'_l
    the kept points and stored bricks of level l before the prune (M, M_l and B_l above are after it), R = min(2^20,
    the bank's pixels) the rays of one visibility batch, and D = 4096 sum_l (B'_l - B_l) the bricks the prune drops,
    the memory held at once beyond the returned grid, the model, the bank and the queries' workspace is at most

        12 M' + D + max(64 P + 28 Q + max_l (8 M'_l + 4096 B'_l),  68 R,  24 max_l M'_l + 4096 max_l B'_l + 2^24,
                        (72 + 12 nc) slab_points + [quantize] 12 nc (max_l M_l + 2^19))

    bytes: the positions and fp32 scores of all kept points, held until the prune, and the pools of the bricks it
    drops; then the structure pass as above; one batch of rays (68 bytes a ray); one level's pool twice while it is
    compacted, with its new row numbers, new positions and the rewrite of 2^10 bricks at a time; and the SH rows of
    the survivors as above."""
    if not 0 <= int(degree) <= 3:
        raise ValueError(f"degree {degree}: need 0..3")
    res = level_resolutions(resolution, levels)
    if not sparse:
        dens = [density_grid(model, r, bounds) for r in res]
        baked, indices, occ = grid_structure(dens, threshold, block)
        if prune is not None:
            # neither the visibility nor the prune reads the rows: degree-0 zero rows stand in for them
            zeros = [torch.zeros(int((i >= 0).sum()), 1, 3, device=i.device) for i in indices]
            rowless = BakedGrid(baked, indices, zeros, occ, bounds, 0, float(model.rgb_padding), block)
            del dens, zeros, baked, indices
            rowless = prune_grid(rowless, prune, weight_threshold)
            baked = [rowless.density(lvl) for lvl in range(len(res))]
            indices = [rowless.index(lvl) for lvl in range(len(res))]
            occ = rowless.occupancy
            del rowless
        sh = [_bake_rows(model, r, (idx.reshape(-1) >= 0).nonzero().reshape(-1), bounds, degree, n_theta, slab_points)
              for r, idx in zip(res, indices)]
        grid = BakedGrid(baked, indices, sh, occ, bounds, degree, float(model.rgb_padding), block)
        return grid.quantize() if quantize else grid
    tx, ty = -(-res[0][0] // BRICK), -(-res[0][1] // BRICK)
    slab = max(1, int(stream_points) // (BRICK ** 3 * ty * tx))
    tables, pools, positions, occ = sparse_grid_structure(
        lambda lvl, z0, z1: density_grid(model, res[lvl], bounds, z_range=(z0, z1)), resolution, levels, threshold,
        block, slab)
    if prune is not None:
        rowless = BakedGrid.from_bricks(tables, pools, res, [torch.empty(0, 1, 3, device=occ.device)] * len(res), occ,
                                        bounds, 0, 0.0, block)
        scores = [torch.zeros(p.numel(), device=occ.device) for p in positions]
        _sweep_bank(rowless, prune, rowless.default_step(), scores)
        del rowless  # _prune_bricks releases the pools level by level
        tables, pools, positions, occ = _prune_bricks(tables, pools, positions, res, scores, weight_threshold, block,
                                                      slab)
    sh, scales, offsets = [], [], []
    for lvl, r in enumerate(res):
        rows = _bake_rows(model, r, positions[lvl], bounds, degree, n_theta, slab_points)
        positions[lvl] = None
        if quantize:
            rows, scale, offset = _quantize_rows(rows, lvl)
            scales.append(scale)
            offsets.append(offset)
        sh.append(rows)
    return BakedGrid.from_bricks(tables, pools, res, sh, occ, bounds, degree, float(model.rgb_padding), block,
                                 scales if quantize else None, offsets if quantize else None)


def _bake_rows(model, resolution, flat: torch.Tensor, bounds, degree: int, n_theta: int,
               slab_points: int) -> torch.Tensor:
    """The raw SH rows [len(flat), (degree + 1)^2, 3] of the lattice points at int64 positions `flat` (x fastest) of
    a level's lattice, `bake_sh(raw=True)` of their voxel Gaussians in calls of `slab_points` points."""
    dev = flat.device
    (xs, ys, zs), _ = lattice_axes(resolution, bounds, dev)
    var = torch.tensor(voxel_variance(resolution, bounds), device=dev)
    out = torch.empty(flat.numel(), (int(degree) + 1) ** 2, 3, device=dev)
    nx, ny = resolution[0], resolution[1]
    for s in range(0, flat.numel(), slab_points):
        p = flat[s:s + slab_points]
        means = torch.stack([xs[p % nx], ys[(p // nx) % ny], zs[p // (nx * ny)]], dim=-1)
        out[s:s + len(p)] = bake_sh(model, means, var.expand(len(p), 3), degree, n_theta, raw=True)
    return out


@torch.no_grad()
def render_baked_frame(grid: BakedGrid, c2w, height: int = 800, width: int = 800, white_bkgd: bool = True,
                       camera_angle_x: float = BLENDER_CAMERA_ANGLE_X, near: float = 2.0, far: float = 6.0,
                       world: int = 1, rank: int = 0, group=None, device=None, step: Optional[float] = None):
    """One frame from a baked grid, with `render.render_frame`'s rays and row sharding: (rgb [H,W,3], distance [H,W],
    acc [H,W]) on every rank."""
    dev = device or grid.device
    r0, r1 = shard_rows(height, world, rank)
    rays = generate_rays(c2w, height, width, camera_angle_x, near, far, rows=(r0, r1), device=dev)
    rgb, dist, acc = grid.render(rays, white_bkgd, step)
    local = torch.cat([rgb, dist[:, None], acc[:, None]], dim=1)  # [rows*W, 5]
    counts = [(shard_rows(height, world, r)[1] - shard_rows(height, world, r)[0]) * width for r in range(world)]
    full = gather_rows(local, counts, group)
    return full[:, 0:3].reshape(height, width, 3), full[:, 3].reshape(height, width), full[:, 4].reshape(height, width)


@torch.no_grad()
def render_proposed_frame(model, grid: BakedGrid, c2w, height: int = 800, width: int = 800, white_bkgd: bool = True,
                          camera_angle_x: float = BLENDER_CAMERA_ANGLE_X, near: float = 2.0, far: float = 6.0,
                          world: int = 1, rank: int = 0, group=None, device=None):
    """One frame of `model.forward_proposed(rays, grid, False, white_bkgd)` (the MLP's fine level, placed by the
    grid's proposal weights), with `render.render_frame`'s rays and row sharding: (fine_rgb [H,W,3], distance [H,W]) on
    every rank."""
    dev = device or next(model.parameters()).device
    r0, r1 = shard_rows(height, world, rank)
    rays = generate_rays(c2w, height, width, camera_angle_x, near, far, rows=(r0, r1), device=dev)
    ret = model.forward_proposed(rays, grid, False, white_bkgd)
    local = torch.cat([ret[-1][0], ret[-1][1][:, None]], dim=1)  # [rows*W, 4]
    counts = [(shard_rows(height, world, r)[1] - shard_rows(height, world, r)[0]) * width for r in range(world)]
    full = gather_rows(local, counts, group)
    return full[:, 0:3].reshape(height, width, 3), full[:, 3].reshape(height, width)


def prune_grid(grid: BakedGrid, bank, weight_threshold: float = DEFAULT_WEIGHT_THRESHOLD, step: Optional[float] = None,
               batch_size: int = 1 << 20) -> BakedGrid:
    """Prune the points no training ray sees (PlenOctrees): `grid.visibility` over every pixel of a `DeviceRayBank`,
    in id order and batches of `batch_size`, then `grid.prune(scores, weight_threshold)`.  Returns the new grid; the
    intended pipeline is `bake_grid` -> `prune_grid` -> `finetune_grid`, at one `step`."""
    if int(batch_size) < 1:
        raise ValueError(f"batch_size {batch_size}: need >= 1")
    scores = [torch.zeros(m, device=grid.device) for m in grid.kept]
    grid._refuse_sparse("visibility")
    grid._refuse_quantized("visibility")
    _sweep_bank(grid, bank, step, scores, batch_size)
    return grid.prune(scores, weight_threshold)


def _sweep_bank(grid: BakedGrid, bank, step: Optional[float], scores: List[torch.Tensor],
                batch_size: int = 1 << 20) -> None:
    """Raise `scores` (per level [M_l] in SH-row order) in place to the visibility scores of every pixel of a
    `DeviceRayBank`, in id order and batches of `batch_size`, on dense cells or bricks (`BakedGrid._visibility`)."""
    for s in range(0, bank.num_pixels, int(batch_size)):
        rays, _ = bank.rays(torch.arange(s, min(s + int(batch_size), bank.num_pixels), device=bank.device))
        grid._visibility(rays, step, scores)


def finetune_grid(grid: BakedGrid, bank, steps: int, batch_size: int = 8192, lr_density: float = FINETUNE_LR_DENSITY,
                  lr_sh: float = FINETUNE_LR_SH, white_bkgd: bool = True, step: Optional[float] = None,
                  generator: Optional[torch.Generator] = None, tv_density: float = 0.0,
                  tv_sh: float = 0.0) -> List[float]:
    """Fine-tune a baked grid's kept densities and SH rows against a `DeviceRayBank`'s pixels (PlenOctrees / SNeRG
    style): per step a random batch, `grid.render`, the MSE against the targets, its backward through the grid ray
    marcher, and one `FusedAdam` step (`lr_density` for the densities, `lr_sh` for the SH rows).  With `tv_density` or
    `tv_sh` > 0 the loss is MSE + tv_density TV_density + tv_sh TV_sh (`BakedGrid.total_variation`, Plenoxels' prior);
    with both 0 nothing else is launched.  Makes the grid trainable if it is not; returns the per-step MSE, without the
    prior, so that runs with different weights compare directly."""
    from .train import FusedAdam
    tv_density, tv_sh = float(tv_density), float(tv_sh)
    if not (tv_density >= 0 and tv_sh >= 0):
        raise ValueError(f"tv_density={tv_density}, tv_sh={tv_sh}: need weights >= 0")
    grid.requires_grad_(True)
    params = [p for p in grid.parameters() if p.numel()]  # a level without kept points has nothing to train
    opt = FusedAdam([{"params": [p for p in params if p.dim() == 1], "lr": float(lr_density)},
                     {"params": [p for p in params if p.dim() == 3], "lr": float(lr_sh)}])
    losses = []
    for _ in range(int(steps)):
        rays, target = bank.sample(batch_size, generator)
        rgb, _, _ = grid.render(rays, white_bkgd, step)
        loss = torch.mean((rgb - target) ** 2)
        total = loss
        if tv_density or tv_sh:
            tv_d, tv_s = grid.total_variation()
            total = loss + tv_density * tv_d + tv_sh * tv_s
        for p in params:
            p.grad = None
        total.backward()
        opt.step()
        losses.append(loss.detach())
    return torch.stack(losses).tolist() if losses else []


def finetune_proposal(grid: BakedGrid, model, bank, steps: int, batch_size: int = 8192,
                      lr_density: float = FINETUNE_LR_DENSITY, generator: Optional[torch.Generator] = None) -> List[float]:
    """Fine-tune a baked grid's kept densities as the proposal of `model` (`MipNerf.forward_proposed`), with mip-NeRF
    360's interlevel loss.  Per step: a random batch of a `DeviceRayBank`'s rays; level 0's randomized fenceposts t_hat
    as `forward_proposed` draws them; the proposal weights w_hat = `grid.proposal(rays, t_hat, differentiable=True)`,
    with their graph; `model`'s later levels from (t_hat, w_hat) under no_grad; `ops.interlevel_loss` of the last
    level's (t, w) against (t_hat, w_hat), its backward through mipnerf_b200_grid_proposal_backward, and one
    `FusedAdam` step (`lr_density`) on the kept densities only.  The SH rows and the kept set never change, and the model is not trained.  The loss
    can raise density only at kept points whose samples fall in occupied macro cells: the proposal weights have no
    gradient in empty space, so fine weight behind a hole the bake left stays uncovered.  Makes the grid trainable if
    it is not, and refuses what `forward_proposed` refuses; returns the per-step losses."""
    from .ops import interlevel_loss
    from .train import FusedAdam
    model._check_proposed("finetune_proposal")
    grid.requires_grad_(True)
    params = [d for d in grid.kept_density if d.numel()]  # a level without kept points has nothing to train
    opt = FusedAdam([{"params": params, "lr": float(lr_density)}])
    losses = []
    for _ in range(int(steps)):
        rays, _ = bank.sample(batch_size, generator)
        t_hat, rng, u_jitter, normals = model._proposal_fenceposts(rays, True, None, None, None)
        w_hat = grid.proposal(rays, t_hat, differentiable=True)
        with torch.no_grad():
            fine = model._forward_from(rays, t_hat, w_hat.detach(), True, True, rng, u_jitter, normals, False)[-1]
        loss = interlevel_loss(fine[4], fine[3], t_hat, w_hat)
        for p in params:
            p.grad = None
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    return torch.stack(losses).tolist() if losses else []
