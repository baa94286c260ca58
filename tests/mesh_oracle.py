"""numpy oracle of the mesh extraction (nsb_mesh_count / nsb_mesh_emit, DESIGN 4.2d): marching tetrahedra on the Kuhn split
with the same vertex and face order.  Written from the definition, not from the kernel: the triangle of each
(tetrahedron, inside pattern) is oriented by integer geometry of the cube corners (the normal of the triangle through
doubled edge midpoints against the direction from the inside corners to the outside ones), not by a parity rule."""
import numpy as np

# edge slots of a grid point: direction (dx, dy, dz)
SLOTS = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]
AXES = [(1, 0, 0), (0, 1, 0), (0, 0, 1)]
PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


def tetrahedra():
    """The 6 tetrahedra of a cell: corners (as integer offsets) 000, e_a, e_a + e_b, 111 per permutation."""
    out = []
    for a, b, _ in PERMS:
        ea, eb = np.array(AXES[a]), np.array(AXES[b])
        out.append([np.zeros(3, int), ea, ea + eb, np.ones(3, int)])
    return out


def _oriented(tri, corners, inside):
    """tri: 3 edges (pairs of tet-corner indices); True when its normal points from the inside corners to the outside."""
    m = [corners[p] + corners[q] for p, q in tri]          # doubled midpoints, integers
    nrm = np.cross(m[1] - m[0], m[2] - m[0])
    ins = [c for c in range(4) if inside[c]]
    outs = [c for c in range(4) if not inside[c]]
    direction = sum(corners[c] for c in outs) * len(ins) - sum(corners[c] for c in ins) * len(outs)
    s = int(np.dot(nrm, direction))
    assert s != 0
    return s > 0


def case_table():
    """table[t][pattern] = list of triangles, each 3 edges (p, q) of tet-corner indices; pattern bit c = corner c inside.
    2 inside corners i < j, outside k < l: the quad (ik, il, jl, jk), or its reverse (ik, jk, jl, il) when that one is
    oriented, fanned from ik."""
    table = []
    for corners in tetrahedra():
        rows = []
        for pattern in range(16):
            inside = [(pattern >> c) & 1 for c in range(4)]
            ins = [c for c in range(4) if inside[c]]
            outs = [c for c in range(4) if not inside[c]]
            tris = []
            if len(ins) in (1, 3):
                lone = ins[0] if len(ins) == 1 else outs[0]
                rest = outs if len(ins) == 1 else ins
                tri = [(lone, rest[0]), (lone, rest[1]), (lone, rest[2])]
                if not _oriented(tri, corners, inside):
                    tri = [tri[0], tri[2], tri[1]]
                tris = [tri]
            elif len(ins) == 2:
                (i, j), (k, l) = ins, outs
                q = [(i, k), (i, l), (j, l), (j, k)]
                if not _oriented(q[:3], corners, inside):
                    q = [(i, k), (j, k), (j, l), (i, l)]
                tris = [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
            rows.append(tris)
        table.append(rows)
    return table


def grid_positions(n, box_min, h):
    """float32 coordinate of index 0..n-1 on one axis: box_min + i * h, rounded after each operation."""
    return np.float32(box_min) + np.arange(n, dtype=np.float32) * np.float32(h)


def marching_tetrahedra(sigma, level, box_min, h):
    """sigma [nz, ny, nx] -> (vertices float32 [V,3], faces int32 [F,3]) in the kernel's order."""
    sigma = np.ascontiguousarray(sigma, dtype=np.float32)
    nz, ny, nx = sigma.shape
    level = np.float32(level)
    inside = sigma > level
    cross = np.zeros((nz, ny, nx, 7), dtype=bool)
    for s, (dx, dy, dz) in enumerate(SLOTS):
        cross[:nz - dz, :ny - dy, :nx - dx, s] = inside[:nz - dz, :ny - dy, :nx - dx] != inside[dz:, dy:, dx:]
    flat = cross.reshape(-1, 7)
    ids = np.full(flat.shape, -1, dtype=np.int64)
    ids[flat] = np.arange(int(flat.sum()))                 # (point, slot) order
    pt, slot = np.nonzero(flat)
    z, rem = np.divmod(pt, nx * ny)
    y, x = np.divmod(rem, nx)
    d = np.array(SLOTS)[slot]
    s0 = sigma.reshape(-1)[pt]
    s1 = sigma[z + d[:, 2], y + d[:, 1], x + d[:, 0]]
    t = (level - s0) / (s1 - s0)
    axes = [grid_positions(n, box_min[k], h[k]) for k, n in enumerate((nx, ny, nz))]
    verts = np.empty((len(pt), 3), dtype=np.float32)
    for k, (i, dk) in enumerate(((x, d[:, 0]), (y, d[:, 1]), (z, d[:, 2]))):
        p0 = axes[k][i]
        p1 = axes[k][np.minimum(i + dk, axes[k].shape[0] - 1)]
        verts[:, k] = p0 + t * (p1 - p0)
    # faces: cells in (z, y, x) order, then tetrahedron, then triangle
    cz, cy, cx = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    cz, cy, cx = cz.reshape(-1), cy.reshape(-1), cx.reshape(-1)
    n_cells = cz.shape[0]
    table = case_table()
    tets = tetrahedra()
    faces = np.full((n_cells, 6, 2, 3), -1, dtype=np.int64)
    used = np.zeros((n_cells, 6, 2), dtype=bool)
    for t, corners in enumerate(tets):
        pattern = np.zeros(n_cells, dtype=np.int64)
        for c, off in enumerate(corners):
            pattern |= inside[cz + off[2], cy + off[1], cx + off[0]].astype(np.int64) << c
        for pat in range(16):
            sel = np.nonzero(pattern == pat)[0]
            if sel.size == 0:
                continue
            for r, tri in enumerate(table[t][pat]):
                used[sel, t, r] = True
                for e, (p, q) in enumerate(tri):
                    lo = np.minimum(corners[p], corners[q])
                    dv = tuple(np.abs(corners[p] - corners[q]))
                    owner = (cx[sel] + lo[0]) + nx * ((cy[sel] + lo[1]) + ny * (cz[sel] + lo[2]))
                    faces[sel, t, r, e] = ids[owner, SLOTS.index(dv)]
    faces = faces[used]
    assert (faces >= 0).all()
    return verts, faces.astype(np.int32)


# ------------------------------------------------------------------ mesh checks
def edge_use(faces):
    """(undirected edges [E,2], how often each is used, how often in the direction lo -> hi)."""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).astype(np.int64)
    fwd = e[:, 0] < e[:, 1]
    key = np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1])
    uniq, inv, counts = np.unique(key, return_inverse=True, return_counts=True)
    n_fwd = np.bincount(inv, weights=fwd, minlength=uniq.shape[0])
    return uniq, counts, n_fwd


def signed_volume(verts, faces):
    v = verts.astype(np.float64)[faces]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def sample_grid(fn, n, lo=-1.0, hi=1.0):
    """fn on an n^3 grid over [lo, hi]^3 -> (sigma [n,n,n] (z, y, x), box_min, h)."""
    h = np.float32((hi - lo) / (n - 1))
    ax = grid_positions(n, lo, h)
    Z, Y, X = np.meshgrid(ax, ax, ax, indexing="ij")
    return fn(X.astype(np.float64), Y.astype(np.float64), Z.astype(np.float64)).astype(np.float32), [lo] * 3, [float(h)] * 3


def sphere(r):
    return lambda X, Y, Z: r - np.sqrt(X * X + Y * Y + Z * Z)


def torus(R, r):
    return lambda X, Y, Z: r - np.sqrt((np.sqrt(X * X + Y * Y) - R) ** 2 + Z * Z)
