"""numpy implementation of the isosurface rules of include/mipnerf_b200.h (marching tetrahedra, Kuhn subdivision), the
checker of the CUDA extractor, and mesh checks (manifoldness, orientation, Euler characteristic, enclosed volume).

The triangle winding is derived here from geometry (the normal of the triangle through the lattice midpoints of its
edges, against the direction from the tetrahedron's inside corners to its outside ones), independently of the CUDA
kernel's table and its orientation-parity rule."""
import itertools

import numpy as np

DIRS = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]  # (dx, dy, dz)
PERMS = list(itertools.permutations(range(3)))          # (x,y,z) (x,z,y) (y,x,z) (y,z,x) (z,x,y) (z,y,x)
TET_EDGES = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def kuhn_corners(perm):
    """The four corner offsets (dx, dy, dz) of the tetrahedron v0 -> v0+e_a -> v0+e_a+e_b -> v0+(1,1,1)."""
    c = [np.zeros(3, dtype=np.int64)]
    for a in perm:
        nxt = c[-1].copy()
        nxt[a] = 1
        c.append(nxt)
    return c


def _triangles(perm, pattern):
    """Triangles (triples of tetrahedron edges) of one tetrahedron for an inside pattern, outward-wound."""
    corners = [c.astype(float) for c in kuhn_corners(perm)]
    ins = [v for v in range(4) if pattern >> v & 1]
    out = [v for v in range(4) if not pattern >> v & 1]
    e = lambda a, b: TET_EDGES.index((min(a, b), max(a, b)))  # noqa: E731
    if len(ins) == 1:
        tris = [[e(ins[0], o) for o in out]]
    elif len(ins) == 3:
        tris = [[e(i, out[0]) for i in ins]]
    elif len(ins) == 2:
        (i, j), (k, l) = ins, out
        tris = [[e(i, k), e(i, l), e(j, l)], [e(i, k), e(j, l), e(j, k)]]
    else:
        return []
    res = []
    for t in tris:
        m = [(corners[TET_EDGES[x][0]] + corners[TET_EDGES[x][1]]) / 2 for x in t]
        n = np.cross(m[1] - m[0], m[2] - m[0])
        d = np.mean([corners[o] for o in out], axis=0) - np.mean([corners[i] for i in ins], axis=0)
        res.append(t if np.dot(n, d) > 0 else [t[0], t[2], t[1]])
    return res


def isosurface(grid, iso, bounds):
    """grid [nz, ny, nx] -> (verts [V,3] float32, faces [F,3] int32, vertex edges [V, 2, 3] lattice (i, j, k) of the
    two ends of each vertex's edge)."""
    g = np.asarray(grid, dtype=np.float32)
    nz, ny, nx = g.shape
    n = np.array([nx, ny, nz])
    lo = np.asarray(bounds[0], dtype=np.float32)
    hi = np.asarray(bounds[1], dtype=np.float32)
    step = (hi - lo) / (n.astype(np.float32) - np.float32(1))
    iso = np.float32(iso)
    inside = g > iso
    kk, jj, ii = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    cross = np.zeros((nz, ny, nx, 7), dtype=bool)
    for d, (dx, dy, dz) in enumerate(DIRS):
        cross[:nz - dz, :ny - dy, :nx - dx, d] = inside[:nz - dz, :ny - dy, :nx - dx] != inside[dz:, dy:, dx:]
    flat = cross.reshape(-1)
    ids = np.full(flat.shape, -1, dtype=np.int64)
    ids[flat] = np.arange(int(flat.sum()))
    ids = ids.reshape(cross.shape)
    # vertices, in id order
    k, j, i, d = np.nonzero(cross)
    dd = np.array(DIRS)[d]
    va = g[k, j, i]
    vb = g[k + dd[:, 2], j + dd[:, 1], i + dd[:, 0]]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (iso - va) / (vb - va)
    t = np.where(np.isnan(t), np.float32(0.5), t).astype(np.float32)
    idx_a = np.stack([i, j, k], axis=1)
    idx_b = idx_a + dd
    pa = lo + idx_a.astype(np.float32) * step
    pb = lo + idx_b.astype(np.float32) * step
    verts = (pa + t[:, None] * (pb - pa)).astype(np.float32)
    edges = np.stack([idx_a, idx_b], axis=1)
    # faces: (cell x-fastest, tetrahedron, triangle)
    cz, cy, cx = nz - 1, ny - 1, nx - 1
    faces = np.full((cz, cy, cx, 6, 2, 3), -1, dtype=np.int64)
    for ti, perm in enumerate(PERMS):
        corners = kuhn_corners(perm)
        ins = [inside[c[2]:c[2] + cz, c[1]:c[1] + cy, c[0]:c[0] + cx] for c in corners]
        pattern = ins[0].astype(int) | ins[1] << 1 | ins[2] << 2 | ins[3] << 3
        for pat in range(16):
            sel = pattern == pat
            if not sel.any():
                continue
            for r, tri in enumerate(_triangles(perm, pat)):
                for q, te in enumerate(tri):
                    ca, cb = corners[TET_EDGES[te][0]], corners[TET_EDGES[te][1]]
                    dvec = tuple(int(v) for v in cb - ca)
                    dir_idx = DIRS.index(dvec)
                    sub = ids[ca[2]:ca[2] + cz, ca[1]:ca[1] + cy, ca[0]:ca[0] + cx, dir_idx]
                    faces[..., ti, r, q][sel] = sub[sel]
    faces = faces.reshape(-1, 3)
    faces = faces[faces[:, 0] >= 0].astype(np.int32)
    return verts, faces, edges


def directed_edge_counts(faces):
    """{(a, b): count} of the directed edges of the faces."""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).astype(np.int64)
    keys, counts = np.unique(e[:, 0] * (1 << 32) + e[:, 1], return_counts=True)
    return dict(zip(((int(k) >> 32, int(k) & 0xFFFFFFFF) for k in keys), counts.tolist()))


def manifold_violations(faces, skip_edge=None):
    """Directed edges that do not appear exactly once with their reverse exactly once (closed, consistently oriented
    2-manifold); `skip_edge(a, b)` excludes edges (on the box faces of an open mesh)."""
    de = directed_edge_counts(faces)
    bad = []
    for (a, b), c in de.items():
        if skip_edge is not None and skip_edge(a, b):
            continue
        if c != 1 or de.get((b, a), 0) != 1:
            bad.append((a, b))
    return bad


def on_box_face(edges, n):
    """skip_edge for a grid of n = (nx, ny, nz) points: both vertices lie on one face of the lattice's box (both ends of
    both vertex edges on the same boundary plane)."""
    n = np.asarray(n)
    lo_planes = (edges == 0).all(axis=1)          # [V, 3]: the vertex's whole edge lies on plane axis = 0
    hi_planes = (edges == n - 1).all(axis=1)

    def skip(a, b):
        return bool((lo_planes[a] & lo_planes[b]).any() or (hi_planes[a] & hi_planes[b]).any())
    return skip


def euler_characteristic(verts, faces):
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).astype(np.int64)
    e = np.sort(e, axis=1)
    num_edges = len(np.unique(e[:, 0] * (1 << 32) + e[:, 1]))
    used = len(np.unique(faces))
    return used - num_edges + len(faces)


def enclosed_volume(verts, faces):
    """Signed volume (divergence theorem): positive when the normals point outwards."""
    v = np.asarray(verts, dtype=np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def read_ply(path):
    """The (verts, faces) of a binary little-endian triangle PLY as mipnerf_pl_b200.write_ply writes it."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")
    assert header[1] == "format binary_little_endian 1.0", header
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    v = np.frombuffer(data, dtype="<f4", count=3 * nv, offset=end).reshape(nv, 3)
    rec = np.frombuffer(data, dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=nf, offset=end + 12 * nv)
    assert (rec["n"] == 3).all() and end + 12 * nv + 13 * nf == len(data)
    return v.copy(), rec["idx"].copy()


def sphere_grid(n, radius, bounds=((-1.0,) * 3, (1.0,) * 3)):
    """radius - |x| on an n^3 lattice (positive inside)."""
    xs = [np.linspace(bounds[0][a], bounds[1][a], n, dtype=np.float64) for a in range(3)]
    z, y, x = np.meshgrid(xs[2], xs[1], xs[0], indexing="ij")
    return (radius - np.sqrt(x * x + y * y + z * z)).astype(np.float32)


def torus_grid(n, big, small, bounds=((-1.0,) * 3, (1.0,) * 3)):
    """small - distance to the circle of radius `big` in the xy plane (positive inside)."""
    xs = [np.linspace(bounds[0][a], bounds[1][a], n, dtype=np.float64) for a in range(3)]
    z, y, x = np.meshgrid(xs[2], xs[1], xs[0], indexing="ij")
    q = np.sqrt(x * x + y * y) - big
    return (small - np.sqrt(q * q + z * z)).astype(np.float32)
