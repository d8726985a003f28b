"""Float64 restatement of the surface extractor's field and float32 restatement of its polygonisation (DESIGN.md section 15).

TEST INFRASTRUCTURE ONLY.
  - `field64`: phi(p) = sum_j V_j W(|p - x_j|) at the lattice points in float64 (pairs from a k-d tree), with the bound its
    float32 evaluation must meet, as ref64.py bounds a gather pass: (n + c) u A + K per point.
  - `polygonise`: the marching-tetrahedra rule of include/sph.h in float32 numpy, operation by operation, so that it
    reproduces the device's vertices bit for bit and its triangles exactly from the same field.  `dtype=np.float64` runs the
    same rule in float64 (the float64 mesh of the volume check).
  - `normals64`: -grad phi / |grad phi| at the vertices in float64 with the bound of grad phi.
  - mesh properties: edge manifoldness, orientation, components, Euler characteristic, enclosed volume and area.
"""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

from oracle.ref64 import C_NORM, U, kernel

F = np.float32
C_FIELD = C_NORM + 3   # V_j W: the product 1, the fma 0, dx 1 (in kerr), margin 1
C_GRAD = C_NORM + 12   # W'(r) / r: the division 1, * V 1, * dx 1 + dx 1, fma 0, g's own 6.2, margin 1.8

# Edge directions a lattice point owns, in vertex order: bit a = axis a
DIR_BITS = (1, 2, 4, 3, 5, 6, 7)
DIR_INDEX = {b: k for k, b in enumerate(DIR_BITS)}
# Kuhn tetrahedra (0, e_a, e_a + e_b, 1), permutations xyz, xzy, yxz, yzx, zxy, zyx: corner offset bits; odd ones flip winding
TETS = ((0, 1, 3, 7), (0, 1, 5, 7), (0, 2, 3, 7), (0, 2, 6, 7), (0, 4, 5, 7), (0, 4, 6, 7))
TET_ODD = (False, True, True, False, False, True)
TET_EDGES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
# case (sum of 2^k over the inside corners k of a positively oriented tetrahedron) -> triangles as tetrahedron edges, wound
# counter-clockwise seen from outside (lower phi)
CASES = (
    (), ((0, 1, 2),), ((0, 4, 3),), ((1, 2, 4), (1, 4, 3)),
    ((1, 3, 5),), ((0, 5, 2), (0, 3, 5)), ((0, 4, 5), (0, 5, 1)), ((2, 4, 5),),
    ((2, 5, 4),), ((0, 1, 5), (0, 5, 4)), ((0, 5, 3), (0, 2, 5)), ((1, 5, 3),),
    ((1, 3, 4), (1, 4, 2)), ((0, 3, 4),), ((0, 2, 1),), (),
)


# ---- lattice -------------------------------------------------------------------------------------------------------------
def default_box(positions, h):
    """The selected fluids' AABB grown by h (float32)."""
    p = np.asarray(positions, F)
    return p.min(axis=0) - F(h), p.max(axis=0) + F(h)


def lattice(lo, hi, spacing):
    """(origin[3], dims[3]): origin = s floor(lo / s), dims = ceil((hi - origin) / s) + 1, in float32."""
    s = F(spacing)
    lo, hi = np.asarray(lo, F), np.asarray(hi, F)
    o = (s * np.floor(lo / s)).astype(F)
    n = (np.ceil((hi - o) / s) + F(1)).astype(np.int64)
    return o, n


def coords(origin, dims, spacing, dtype=F):
    """Per-axis point coordinates origin + (float)i * spacing: a rounded product, then a rounded sum."""
    s = F(spacing)
    return [(F(origin[a]) + (np.arange(dims[a]).astype(F) * s).astype(F)).astype(F).astype(dtype) for a in range(3)]


def points(origin, dims, spacing):
    """All lattice points, x fastest, float32 [n, 3]."""
    cx, cy, cz = coords(origin, dims, spacing)
    Z, Y, X = np.meshgrid(cz, cy, cx, indexing="ij")
    return np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1)


# ---- field ---------------------------------------------------------------------------------------------------------------
def field64(positions, volumes, pts, h, kind=0):
    """(phi, bound) in float64 at the float32 points pts[n, 3]: phi = sum_j V_j W(|p - x_j|) over the pairs within h."""
    x = np.asarray(positions, F).astype(np.float64)
    v = np.broadcast_to(np.asarray(volumes, F).astype(np.float64), (len(x),))
    p = np.asarray(pts, F).astype(np.float64)
    phi = np.zeros(len(p))
    A = np.zeros(len(p))
    K = np.zeros(len(p))
    n = np.zeros(len(p))
    if len(x) == 0 or len(p) == 0:
        return phi, np.zeros(len(p))
    tree = cKDTree(x)
    step = 1 << 16
    for b in range(0, len(p), step):
        lists = tree.query_ball_point(p[b:b + step], h * (1.0 + 1e-5))
        cnt = np.fromiter((len(l) for l in lists), np.int64, len(lists))
        if not cnt.sum():
            continue
        i = np.repeat(np.arange(b, b + len(lists)), cnt)
        j = np.concatenate([np.asarray(l, np.int64) for l in lists if len(l)])
        r = np.sqrt(((p[i] - x[j]) ** 2).sum(axis=1))
        f, fa, kerr = kernel(kind, "w", r, h)
        np.add.at(phi, i, v[j] * f)
        np.add.at(A, i, v[j] * fa)
        np.add.at(K, i, v[j] * kerr)
        n[b:b + len(lists)] += cnt
    return phi, (n + C_FIELD) * U * A + K


def grad64(positions, volumes, pts, h, kind=0):
    """(grad phi [n, 3], bound per component) in float64 at the float32 points."""
    x = np.asarray(positions, F).astype(np.float64)
    v = np.broadcast_to(np.asarray(volumes, F).astype(np.float64), (len(x),))
    p = np.asarray(pts, F).astype(np.float64)
    g = np.zeros((len(p), 3))
    A = np.zeros(len(p))
    K = np.zeros(len(p))
    n = np.zeros(len(p))
    if len(x) == 0 or len(p) == 0:
        return g, np.zeros(len(p))
    tree = cKDTree(x)
    lists = tree.query_ball_point(p, h * (1.0 + 1e-5))
    cnt = np.fromiter((len(l) for l in lists), np.int64, len(lists))
    if cnt.sum():
        i = np.repeat(np.arange(len(p)), cnt)
        j = np.concatenate([np.asarray(l, np.int64) for l in lists if len(l)])
        dx = p[i] - x[j]
        r = np.sqrt((dx * dx).sum(axis=1))
        f, fa, kerr = kernel(kind, "g", r, h)
        np.add.at(g, i, (v[j] * f)[:, None] * dx)
        np.add.at(A, i, v[j] * fa * r)
        np.add.at(K, i, v[j] * kerr * r)
        n += cnt
    return g, (n + C_GRAD) * U * A + K


def normals64(positions, volumes, verts, h, kind=0):
    """(n = -grad phi / |grad phi|, |grad phi|, bound of each component of grad phi) at the vertices."""
    g, gb = grad64(positions, volumes, verts, h, kind)
    m = np.sqrt((g * g).sum(axis=1))
    nrm = np.where(m[:, None] > 0, -g / np.where(m > 0, m, 1.0)[:, None], 0.0)
    return nrm, m, gb


# ---- polygonisation ------------------------------------------------------------------------------------------------------
def polygonise(phi, origin, dims, spacing, iso, dtype=F, split=None, flip_case=None, t_from_outside=False, tie_outside=False,
               edge_major=False):
    """Vertices [nv, 3] and triangles [nt, 3] (uint32) of phi = iso by the rule of include/sph.h.  phi is flat or
    [nz, ny, nx], x fastest.  The keyword arguments after dtype inject the bugs the tests must catch (mutants): split =
    a cube index cut along the other diagonal (0..6 instead of 7..0), flip_case = a case whose winding is reversed,
    t_from_outside = t measured from the outside end, tie_outside = phi == iso counted as outside, edge_major = vertices
    ordered by edge direction before point."""
    nx, ny, nz = (int(d) for d in dims)
    phi = np.asarray(phi).reshape(-1).astype(dtype)
    iso = dtype(iso)
    npts = nx * ny * nz
    inside = (phi > iso) if tie_outside else (phi >= iso)
    idx = np.arange(npts, dtype=np.int64)
    i, j, k = idx % nx, (idx // nx) % ny, idx // (nx * ny)
    cx, cy, cz = coords(origin, dims, spacing, dtype)

    def nb(b):  # (valid, neighbour index) of the corner with offset bits b
        bx, by, bz = b & 1, (b >> 1) & 1, (b >> 2) & 1
        ok = (i + bx < nx) & (j + by < ny) & (k + bz < nz)
        return ok, idx + bx + nx * (by + ny * bz)

    vid = np.full((npts, 7), -1, np.int64)
    owners, dirs = [], []
    for d, b in enumerate(DIR_BITS):
        ok, q = nb(b)
        q = np.where(ok, q, 0)
        cross = ok & (inside != inside[q])
        owners.append(idx[cross])
        dirs.append(np.full(int(cross.sum()), d))
    owners, dirs = np.concatenate(owners), np.concatenate(dirs)
    order = np.lexsort((owners, dirs)) if edge_major else np.lexsort((dirs, owners))
    owners, dirs = owners[order], dirs[order]
    vid[owners, dirs] = np.arange(len(owners))
    bits = np.asarray(DIR_BITS)[dirs]
    q = owners + (bits & 1) + nx * (((bits >> 1) & 1) + ny * ((bits >> 2) & 1))
    oi, oj, ok_ = owners % nx, (owners // nx) % ny, owners // (nx * ny)
    pa = np.stack([cx[oi], cy[oj], cz[ok_]], axis=1)
    pb = np.stack([cx[oi + (bits & 1)], cy[oj + ((bits >> 1) & 1)], cz[ok_ + ((bits >> 2) & 1)]], axis=1)
    a_is_p = inside[owners]
    fa = np.where(a_is_p, phi[owners], phi[q]).astype(dtype)
    fb = np.where(a_is_p, phi[q], phi[owners]).astype(dtype)
    if t_from_outside:  # the mutant: t of the inside end, applied from the outside end
        a_is_p = ~a_is_p
    xa = np.where(a_is_p[:, None], pa, pb)
    xb = np.where(a_is_p[:, None], pb, pa)
    t = ((iso - fa).astype(dtype) / (fb - fa).astype(dtype)).astype(dtype)
    verts = (xa + (t[:, None] * (xb - xa).astype(dtype)).astype(dtype)).astype(dtype)

    # triangles: cubes are the points with a neighbour on every axis
    cube = idx[(i + 1 < nx) & (j + 1 < ny) & (k + 1 < nz)]
    if not len(cube):
        return verts, np.zeros((0, 3), np.uint32)
    cin = np.zeros((len(cube), 8), bool)
    for b in range(8):
        cin[:, b] = inside[cube + (b & 1) + nx * (((b >> 1) & 1) + ny * ((b >> 2) & 1))]
    tris = []
    keys = []
    for t_, tet in enumerate(TETS):
        case = np.zeros(len(cube), np.int64)
        for v, c in enumerate(tet):
            case |= cin[:, c].astype(np.int64) << v
        for c_ in range(1, 15):
            sel = case == c_
            if not sel.any():
                continue
            for r, tri in enumerate(CASES[c_]):
                ids = []
                for te in tri:
                    cu, cv = tet[TET_EDGES[te][0]], tet[TET_EDGES[te][1]]
                    owner = cube[sel] + (cu & 1) + nx * (((cu >> 1) & 1) + ny * ((cu >> 2) & 1))
                    ids.append(vid[owner, DIR_INDEX[cv ^ cu]])
                if TET_ODD[t_] != (flip_case == c_):
                    ids[1], ids[2] = ids[2], ids[1]
                tris.append(np.stack(ids, axis=1))
                keys.append(cube[sel] * 12 + t_ * 2 + r)
    if split is not None:  # the mutant: one cube cut along the other diagonal (corner 1..6 instead of 0..7)
        tris, keys = _resplit(tris, keys, split, cin, cube, nx, ny, vid, len(verts))
    if not tris:
        return verts, np.zeros((0, 3), np.uint32)
    tris, keys = np.concatenate(tris), np.concatenate(keys)
    tris = tris[np.argsort(keys, kind="stable")]
    return verts, tris.astype(np.uint32)


def _resplit(tris, keys, split, cin, cube, nx, ny, vid, nv):
    """Replaces the triangles of cube `split` by those of the Kuhn split along its other main diagonal (corner offset bits
    reflected in x: 1 .. 6).  Its face diagonals are not the lattice's owned edges: each gets a vertex of its own, numbered
    from nv, as an extractor with the wrong split table would make."""
    sel = [~(kk // 12 == split) for kk in keys]
    tris = [t[s] for t, s in zip(tris, sel)]
    keys = [kk[s] for kk, s in zip(keys, sel)]
    hit = np.nonzero(cube == split)[0]
    extra = {}
    if not len(hit):
        return tris, keys
    c = int(hit[0])
    for t_, tet in enumerate(TETS):
        rt = tuple(b ^ 1 for b in tet)
        case = sum(int(cin[c, b]) << v for v, b in enumerate(rt))
        for r, tri in enumerate(CASES[case]):
            ids = []
            for te in tri:
                cu, cv = rt[TET_EDGES[te][0]], rt[TET_EDGES[te][1]]
                if cu & cv == cu or cu & cv == cv:
                    lo_, hi_ = min(cu, cv, key=lambda b: bin(b).count("1")), max(cu, cv, key=lambda b: bin(b).count("1"))
                    owner = split + (lo_ & 1) + nx * (((lo_ >> 1) & 1) + ny * ((lo_ >> 2) & 1))
                    ids.append(vid[owner, DIR_INDEX[hi_ ^ lo_]])
                else:
                    ids.append(extra.setdefault((min(cu, cv), max(cu, cv)), nv + len(extra)))
            if not TET_ODD[t_]:  # the reflection reverses orientation
                ids[1], ids[2] = ids[2], ids[1]
            tris.append(np.asarray([ids], np.int64))
            keys.append(np.asarray([split * 12 + t_ * 2 + r]))
    return tris, keys


# ---- mesh properties -----------------------------------------------------------------------------------------------------
def edge_counts(tris):
    """(undirected edge -> triangle count, directed edge -> count) as arrays of counts."""
    t = np.asarray(tris, np.int64)
    d = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    m = int(d.max()) + 1 if len(d) else 1
    dk = d[:, 0] * m + d[:, 1]
    uk = np.minimum(d[:, 0], d[:, 1]) * m + np.maximum(d[:, 0], d[:, 1])
    _, uc = np.unique(uk, return_counts=True)
    _, dc = np.unique(dk, return_counts=True)
    return uc, dc


def watertight_oriented(tris):
    """Every undirected edge in exactly two triangles and every directed edge once."""
    uc, dc = edge_counts(tris)
    return bool(np.all(uc == 2) and np.all(dc == 1))


def components(nv, tris):
    t = np.asarray(tris, np.int64)
    if not len(t):
        return 0
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]]])
    g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(nv, nv))
    n, lab = connected_components(g, directed=False)
    return len(np.unique(lab[np.unique(t)]))


def euler(nv, tris):
    """V - E + F over the vertices the triangles use."""
    t = np.asarray(tris, np.int64)
    uc, _ = edge_counts(t)
    return len(np.unique(t)) - len(uc) + len(t)


def volume(verts, tris):
    """Enclosed volume (divergence theorem; positive for outward winding) in float64."""
    v = np.asarray(verts, np.float64)
    t = np.asarray(tris, np.int64)
    if not len(t):
        return 0.0
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def area(verts, tris):
    v = np.asarray(verts, np.float64)
    t = np.asarray(tris, np.int64)
    if not len(t):
        return 0.0
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    return float(0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum())


def volume_bound(phi32, phi64, bound, dims, spacing, iso, mesh_area):
    """How far the enclosed volume of the float32 mesh may lie from that of the float64 mesh: each vertex moves along its
    edge by at most spacing (|e_a| + |e_b|) / |phi_b - phi_a| (e the field's bound), a surface of area A sweeps at most A
    times the largest such move; and every lattice point whose phi lies within its bound of iso may change side, which
    changes the volume of its 8 cubes at most."""
    nx, ny, nz = (int(d) for d in dims)
    p64 = np.asarray(phi64, np.float64).reshape(-1)
    e = np.asarray(bound, np.float64).reshape(-1) + np.abs(np.asarray(phi32, np.float64).reshape(-1) - p64)
    ambiguous = np.abs(p64 - iso) <= e
    worst = 0.0
    idx = np.arange(nx * ny * nz)
    i, j, k = idx % nx, (idx // nx) % ny, idx // (nx * ny)
    for b in DIR_BITS:
        bx, by, bz = b & 1, (b >> 1) & 1, (b >> 2) & 1
        ok = (i + bx < nx) & (j + by < ny) & (k + bz < nz)
        q = np.where(ok, idx + bx + nx * (by + ny * bz), 0)
        cross = ok & ((p64 >= iso) != (p64[q] >= iso)) & ~ambiguous & ~ambiguous[q]
        if cross.any():
            worst = max(worst, float(np.max((e[cross] + e[q[cross]]) / np.abs(p64[q[cross]] - p64[cross]))) * np.sqrt(bx + by + bz))
    return mesh_area * worst * spacing + 8.0 * float(ambiguous.sum()) * spacing ** 3
