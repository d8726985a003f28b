"""Float64 restatement of a parry HeightField as a collider shape: DynamicContactSampling (fluids_pipeline.rs:192-255) and
particles_intersecting_shape (liquid_world.rs:246-281), as DESIGN.md sections 10 and 11 state them, each output with a bound
on the device's float32 evaluation.

TEST INFRASTRUCTURE ONLY.  Written from the contract, not from salva_b200/contact_sampling.py (the float32 restatement the
device is held to bit for bit): that one is checked against this one.  It extends oracle/ref64_colliders.py, whose helpers,
bounds and candidate rules it reuses for the other shapes.

Projection.  parry's literal loop: every triangle of the field, in parry's order (cells column-major, row index fastest,
(p00, p10, p01) before (p10, p11, p01)), each projected as a closed triangle (Ericson's vertex, edge and face regions), the
strictly smaller distance winning and an exact tie going to the earlier triangle.  is_inside is always false.  Vertex x and z
are the contract's float32 grid values (smp_grid); y = h sy is taken in float64.

Bounds.  One rounding per operation of hf_tri (u = 2^-24, relative to the operands' magnitudes) on top of the local point's
bound e_l and the vertex heights' rounding u |y|: differences carry u |x|, a dot product 3 u |a| |b| plus its operands'
bounds, the region products and the edge / face ratios their operands' relative bounds.  The projection carries
e_q = e_l + (the rounding of its formula).  The distance carries e_l, the vertices' and the final additions' rounding,
and only the square of the ratios' error over the distance: they move q along the edge or in the face plane, normal to
p - q, which leaves the distance unchanged to first order.

Near ties.  Where another triangle's distance lies within the bounds of the nearest one's (an exact float64 tie is decided
by parry's order instead), the device may return either projection.  Two nearly coplanar triangles (the two halves of a
smooth cell) tie over a band 1 / angle times wider than the bounds, but their projections differ by only distance x angle:
so the bound of q grows to cover every near-tied projection while their spread stays under TIE_SPREAD of the field's
size (sx / 2 + sz / 2 + max |y|), and the particle is excluded beyond it.

Exclusions (counted per reason).  A particle is excluded from the collider when the nearest-triangle choice lies within the
bounds between triangles whose projections spread further than that, when a region test of Ericson's chain on the winning triangle lies within its bound, when depth lies within its
bound of 1.5 h, and at the AABB and cell-box gates (as ref64_colliders).

`mutant=` applies one plausible bug to the reference: a bound that passes it is too loose.
"""
import numpy as np

from oracle import ref64_colliders as rc

F = np.float32
U = rc.U
G = rc.G
HEIGHTFIELD = 4
TIE_SPREAD = 2.0 ** -10  # a near tie whose projections lie within this fraction of the field's size widens the bound instead
MUTANTS = ("rows_cols_swapped", "other_diagonal", "unscaled_heights", "uncentred_aabb", "is_inside", "local_point_velocity")


def grid32(j, last, half, d):
    """smp_grid in float32: the contract's vertex coordinate."""
    j = np.asarray(j)
    return np.where(j == last, half, -half + j.astype(F) * d).astype(F).astype(np.float64)


def field(heights, scale, mutant=None):
    """All triangles of the field in parry's order: (a, b, c) vertex arrays (T, 3) float64, the vertex y bounds (T, 3)."""
    H = np.asarray(heights, F)
    sx, sy, sz = (F(s) for s in scale)
    nr, nc = H.shape
    hx, hz = sx * F(0.5), sz * F(0.5)
    dx, dz = sx / F(nc - 1), sz / F(nr - 1)
    ni, nj = nr - 1, nc - 1
    J, I = np.meshgrid(np.arange(nj), np.arange(ni), indexing="ij")  # column-major: the row index fastest
    I, J = I.ravel(), J.ravel()
    syf = 1.0 if mutant == "unscaled_heights" else float(sy)

    def vert(i, j):
        if mutant == "rows_cols_swapped":
            x = grid32(i, ni, hx, F(sx / F(ni)))
            z = grid32(j, nj, hz, F(sz / F(nj)))
        else:
            x, z = grid32(j, nj, hx, dx), grid32(i, ni, hz, dz)
        return np.stack([x, H[i, j].astype(np.float64) * syf, z], -1)

    p00, p10, p01, p11 = vert(I, J), vert(I, J + 1), vert(I + 1, J), vert(I + 1, J + 1)
    if mutant == "other_diagonal":
        t0, t1 = (p00, p10, p11), (p00, p11, p01)
    else:
        t0, t1 = (p00, p10, p01), (p10, p11, p01)
    tri = [np.stack([t0[k], t1[k]], 1).reshape(-1, 3) for k in range(3)]
    ylo, yhi = float(H.min()) * float(sy), float(H.max()) * float(sy)
    return dict(a=tri[0], b=tri[1], c=tri[2], ylo=ylo, yhi=yhi, hx=float(hx), hz=float(hz), H=H, sy=float(sy), scale=(sx, sy, sz))


def _dot(x, y):
    return np.sum(x * y, axis=-1)


def _n(x):
    return np.linalg.norm(x, axis=-1)


def _cmp(x, e, le=True):
    """Three-valued x <= 0 (le) or x >= 0: 1 sure true, 0 sure false, -1 within the bound."""
    s = x if le else -x
    return np.where(s < -e, 1, np.where(s > e, 0, np.where(e == 0, (s <= 0).astype(int), -1)))


def _and(*c):
    c = np.stack(c)
    return np.where(np.any(c == 0, axis=0), 0, np.where(np.all(c == 1, axis=0), 1, -1))


def tri64(p, el, a, b, c):
    """Ericson's closest point of the closed triangles (a, b, c) to p (broadcast (..., 3)), with the bound of the device's
    float32 evaluation.  el: the bound of p (norm, (...)).  Returns q, e_q, D = |p - q|, e_D, region (0-6), region_amb."""
    ya, yb, yc = (U * np.abs(v[..., 1]) for v in (a, b, c))
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    e_ab, e_ac = ya + yb + U * _n(ab), ya + yc + U * _n(ac)
    e_ap, e_bp, e_cp = el + ya + U * _n(ap), el + yb + U * _n(bp), el + yc + U * _n(cp)

    def dot(x, ex, y, ey):
        v = _dot(x, y)
        return v, _n(x) * ey + _n(y) * ex + 3 * G * U * _n(x) * _n(y)

    d1, e1 = dot(ab, e_ab, ap, e_ap)
    d2, e2 = dot(ac, e_ac, ap, e_ap)
    d3, e3 = dot(ab, e_ab, bp, e_bp)
    d4, e4 = dot(ac, e_ac, bp, e_bp)
    d5, e5 = dot(ab, e_ab, cp, e_cp)
    d6, e6 = dot(ac, e_ac, cp, e_cp)

    def det(x, ex, y, ey, z, ez, w, ew):  # x y - z w
        v = x * y - z * w
        return v, np.abs(x) * ey + np.abs(y) * ex + np.abs(z) * ew + np.abs(w) * ez + 3 * G * U * (np.abs(x * y) + np.abs(z * w))

    vc, evc = det(d1, e1, d4, e4, d3, e3, d2, e2)
    vb, evb = det(d5, e5, d2, e2, d1, e1, d6, e6)
    va, eva = det(d3, e3, d6, e6, d5, e5, d4, e4)
    e43, ee43 = d4 - d3, e4 + e3 + U * np.abs(d4 - d3)
    e56, ee56 = d5 - d6, e5 + e6 + U * np.abs(d5 - d6)
    tests = [_and(_cmp(d1, e1), _cmp(d2, e2)), _and(_cmp(d3, e3, False), _cmp(d4 - d3, e4 + e3)),
             _and(_cmp(vc, evc), _cmp(d1, e1, False), _cmp(d3, e3)), _and(_cmp(d6, e6, False), _cmp(d5 - d6, e5 + e6)),
             _and(_cmp(vb, evb), _cmp(d2, e2, False), _cmp(d6, e6)), _and(_cmp(va, eva), _cmp(e43, ee43, False), _cmp(e56, ee56, False))]
    ex_tests = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
                (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)]
    region = np.select(ex_tests, np.arange(6), 6)
    amb = np.zeros(region.shape, bool)
    decided = np.zeros(region.shape, bool)
    for t in tests:  # Ericson's chain: every test before the region must be surely false, its own surely true
        amb |= ~decided & (t == -1)
        decided |= t == 1
    with np.errstate(divide="ignore", invalid="ignore"):
        v3 = d1 / (d1 - d3)
        ev3 = (e1 + np.abs(v3) * (e1 + e3)) / np.abs(d1 - d3) + 2 * U * np.abs(v3)
        v5 = d2 / (d2 - d6)
        ev5 = (e2 + np.abs(v5) * (e2 + e6)) / np.abs(d2 - d6) + 2 * U * np.abs(v5)
        v6 = e43 / (e43 + e56)
        ev6 = (ee43 + np.abs(v6) * (ee43 + ee56)) / np.abs(e43 + e56) + 2 * U * np.abs(v6)
        den = (va + vb) + vc
        eden = eva + evb + evc + 2 * U * np.abs(den)
        vf, wf = vb / den, vc / den
        evf = (evb + np.abs(vf) * eden) / np.abs(den) + 3 * U * np.abs(vf)
        ewf = (evc + np.abs(wf) * eden) / np.abs(den) + 3 * U * np.abs(wf)
    cb = c - b
    e_cb = yb + yc + U * _n(cb)
    na = _n(a)
    # per region: q, the bound of its ratios (along the edge or in the face plane) and of its final additions and vertices
    cand = [(a, 0.0, ya), (b, 0.0, yb),
            (a + v3[..., None] * ab, _n(ab) * ev3 + np.abs(v3) * e_ab, ya + yb + 2 * G * U * (na + _n(ab) * np.abs(v3))),
            (c, 0.0, yc),
            (a + v5[..., None] * ac, _n(ac) * ev5 + np.abs(v5) * e_ac, ya + yc + 2 * G * U * (na + _n(ac) * np.abs(v5))),
            (b + v6[..., None] * cb, _n(cb) * ev6 + np.abs(v6) * e_cb, yb + yc + 2 * G * U * (_n(b) + _n(cb) * np.abs(v6))),
            (a + ab * vf[..., None] + ac * wf[..., None], _n(ab) * evf + _n(ac) * ewf + np.abs(vf) * e_ab + np.abs(wf) * e_ac,
             ya + yb + yc + 4 * G * U * (na + _n(ab) * np.abs(vf) + _n(ac) * np.abs(wf)))]
    sel = [region == k for k in range(7)]
    q = np.select([m[..., None] for m in sel], [x for x, _, _ in cand])
    et = np.select(sel, [np.broadcast_to(e, region.shape) for _, e, _ in cand])
    en = np.select(sel, [np.broadcast_to(e, region.shape) for _, _, e in cand])
    eq = el + et + en
    D = _n(p - q)
    # the ratios move q along the edge or in the face plane, where p - q is normal: they change the distance only to second
    # order; the vertices' heights, the final additions, p and the distance's own evaluation change it to first order
    with np.errstate(divide="ignore", invalid="ignore"):
        eD = el + en + np.where(D > 0, (et + en) ** 2 / np.where(D > 0, D, 1.0), et + en) + 3 * G * U * D
    return q, eq, D, eD, region, amb


def project64(fld, l, el, chunk=64):
    """project_local_point over every triangle: q (n, 3), e_q (n,), D (n,), e_D (n,), the winning triangle (n,), and the
    exclusions: the nearest-triangle choice and the region within the winner."""
    l = np.asarray(l, np.float64)
    n = len(l)
    el = np.broadcast_to(np.asarray(el, np.float64), (n,))
    q, eq, D, eD = np.zeros((n, 3)), np.zeros(n), np.zeros(n), np.zeros(n)
    win, amb_choice, amb_region = np.zeros(n, np.int64), np.zeros(n, bool), np.zeros(n, bool)
    A, B, Cv = fld["a"], fld["b"], fld["c"]
    tau = TIE_SPREAD * (fld["hx"] + fld["hz"] + max(abs(fld["ylo"]), abs(fld["yhi"])))
    lo, hi = np.minimum(np.minimum(A, B), Cv), np.maximum(np.maximum(A, B), Cv)
    for s in range(0, n, chunk):
        p = l[s:s + chunk, None, :]
        e = el[s:s + chunk, None]
        # every triangle whose box lies within the nearest vertex's distance (plus slack): the others are farther than a
        # vertex of the field, so they can neither win nor tie, and skipping them leaves the loop's result unchanged
        lb = np.linalg.norm(np.maximum(np.maximum(lo[None] - p, p - hi[None]), 0.0), axis=-1)
        ub = np.linalg.norm(A[None] - p, axis=-1).min(axis=1)
        keep = np.nonzero(np.any(lb <= (ub * (1 + 1e-6) + 1e-6 * (1 + np.abs(p).max()))[:, None], axis=0))[0]
        a, b, c = A[keep][None], B[keep][None], Cv[keep][None]
        Q, EQ, DD, ED, _, AMB = tri64(p, e, a, b, c)
        w = DD.argmin(axis=1)  # the first minimum: parry's order on an exact tie (keep is ascending)
        r = np.arange(len(w))
        dq = np.linalg.norm(Q - Q[r, w][:, None], axis=-1)
        tied = (DD - ED <= (DD[r, w] + ED[r, w])[:, None]) & (DD != DD[r, w][:, None])
        spread = np.where(tied, dq + EQ, 0.0).max(axis=1)  # the device may return any near-tied triangle's projection
        q[s:s + chunk], eq[s:s + chunk], D[s:s + chunk], eD[s:s + chunk] = Q[r, w], np.maximum(EQ[r, w], spread), DD[r, w], ED[r, w]
        win[s:s + chunk], amb_choice[s:s + chunk], amb_region[s:s + chunk] = keep[w], spread > tau, AMB[r, w]
    return q, eq, D, eD, win, amb_choice, amb_region


def surface_below(fld, l):
    """Whether each local point lies below the surface over the footprint (the is_inside mutant)."""
    H, (sx, sy, sz) = fld["H"], fld["scale"]
    nr, nc = H.shape
    x, z = l[:, 0], l[:, 2]
    ok = (np.abs(x) <= sx / 2) & (np.abs(z) <= sz / 2)
    u = np.clip((x + sx / 2) / (sx / (nc - 1)), 0, nc - 1 - 1e-9)
    v = np.clip((z + sz / 2) / (sz / (nr - 1)), 0, nr - 1 - 1e-9)
    j, i = np.floor(u).astype(int), np.floor(v).astype(int)
    fu, fv = u - j, v - i
    h00, h10, h01, h11 = H[i, j], H[i, j + 1], H[i + 1, j], H[i + 1, j + 1]
    y = np.where(fu + fv <= 1, h00 + fu * (h10 - h00) + fv * (h01 - h00), h11 + (1 - fu) * (h01 - h11) + (1 - fv) * (h10 - h11)) * sy
    return ok & (l[:, 1] < y)


def posed_aabb64(fld, R, t, mutant=None):
    """compute_aabb(pos) = Aabb::transform_by: centre R c + t, half extents |R| e."""
    cy, ey = (fld["ylo"] + fld["yhi"]) / 2, (fld["yhi"] - fld["ylo"]) / 2
    e = np.array([fld["hx"], ey, fld["hz"]])
    c = t if mutant == "uncentred_aabb" else R @ np.array([0.0, cy, 0.0]) + t
    ext = np.abs(R) @ e
    return c, ext


def contact64(pos, vel, colliders, dt, h, r, mutant=None):
    """update_boundaries over colliders in slot order, heightfields (kind 4, with heights and scale) among ball / cuboid /
    capsule colliders (ref64_colliders.contact64).  A heightfield never pushes, so each one sees the state the
    non-heightfield colliders before it left.  Returns a ref64_colliders.Contact (samples per collider, pos, vel, bounds,
    excluded) with res.reasons counting the exclusions."""
    N = len(pos)
    others = [k for k, col in enumerate(colliders) if col["kind"] != HEIGHTFIELD]
    res = rc.contact64(pos, vel, [colliders[k] for k in others], dt, h, r,
                       mutant=mutant if mutant in ("local_point_velocity",) else None)
    samples = [None] * len(colliders)
    for j, k in enumerate(others):
        samples[k] = res.samples[j]
    excluded = res.excluded.copy()
    res.hf_candidates = 0
    P0 = rc._f64(pos)
    hh = float(F(h))
    cut = 1.5 * hh
    dtp = float(F(dt))
    c_lo, c_hi = rc._cell_range(P0, hh)
    for k, col in enumerate(colliders):
        if col["kind"] != HEIGHTFIELD:
            continue
        prefix = [colliders[m] for m in range(k) if colliders[m]["kind"] != HEIGHTFIELD]
        pre = rc.contact64(pos, vel, prefix, dt, h, r) if prefix else None
        p, v = (pre.pos, pre.vel) if pre else (rc._f64(pos), rc._f64(vel))
        ep, ev = (pre.ep, pre.ev) if pre else (np.zeros((N, 3)), np.zeros((N, 3)))
        R = rc._f64(col.get("rotation", np.eye(3))).reshape(3, 3)
        t = rc._f64(col.get("translation", (0, 0, 0)))
        perm = rc._signed_perm(R)
        fld = field(col["heights"], col["scale"], mutant)
        cen, ext = posed_aabb64(fld, R, t, mutant)
        mins, maxs = cen - ext - cut, cen + ext + cut
        e_box = G * U * (3 * ext + 2 * (np.abs(cen) + ext + cut) + cut + np.abs(R) @ np.array([0, abs(fld["ylo"]) + abs(fld["yhi"]), 0]))
        lo_q, hi_q = mins / hh, maxs / hh
        lo_tol, hi_tol = e_box / hh + G * U * np.abs(lo_q), e_box / hh + G * U * np.abs(hi_q)
        klo = (np.floor(lo_q - lo_tol), np.floor(lo_q + lo_tol))
        khi = (np.floor(hi_q - hi_tol), np.floor(hi_q + hi_tol))
        sure_in = np.all((c_lo >= klo[1]) & (c_hi <= khi[0]), axis=1)
        sure_out = np.any((c_hi < klo[0]) | (c_lo > khi[1]), axis=1)
        in_box = np.all((np.floor(P0 / hh) >= np.floor(lo_q)) & (np.floor(P0 / hh) <= np.floor(hi_q)), axis=1)
        pr_all = p + v * dtp
        known = np.all((ep == 0) & (ev == 0), axis=1)
        f32 = (p.astype(F) + v.astype(F) * F(dtp)).astype(np.float64)
        e_gen = ep + ev * dtp + G * U * (2 * np.abs(v) * dtp + np.abs(p))
        e_pr_all = np.where(known[:, None], np.abs(f32 - pr_all), e_gen)
        s_box = np.minimum(pr_all - mins, maxs - pr_all)
        tol_box = e_pr_all + e_box
        aabb = np.all(s_box >= 0, axis=1)
        maybe = ~sure_out & ~np.any(s_box < -tol_box, axis=1)
        gate_amb = (~sure_in | ~np.all(s_box > tol_box, axis=1)) & maybe
        res.reasons["cell_or_aabb"] = res.reasons.get("cell_or_aabb", 0) + int((gate_amb & ~excluded).sum())
        excluded |= gate_amb
        res.hf_candidates += int(in_box.sum())
        idx = np.nonzero(in_box & aabb)[0]
        amb_extra = np.nonzero(~sure_out & excluded & ~(in_box & aabb))[0]
        pr, e_pr = pr_all[idx], e_pr_all[idx]
        w = pr - t
        e_w = rc._rn(w, e_pr)
        l = w @ R
        e_l = e_w @ np.abs(R)
        if not perm:
            e_l = e_l + G * 3 * U * (np.abs(w) @ np.abs(R))
        q, eq, D, eD, _, amb_choice, amb_region = project64(fld, l, np.linalg.norm(e_l, axis=1))
        qw = q @ R.T + t
        e_qw = eq[:, None] * np.ones(3) + G * U * np.abs(qw)
        if not perm:
            e_qw = e_qw + G * 3 * U * (np.abs(q) @ np.abs(R).T)
        d = pr - qw
        depth = np.linalg.norm(d, axis=1)
        e_depth = np.linalg.norm(e_pr + e_qw, axis=1) + 3 * G * U * depth
        beyond = depth > cut
        amb_cut = rc._near(depth - cut, e_depth + U * cut)
        for name, m in (("triangle_choice", amb_choice), ("region", amb_region), ("depth_cut", amb_cut & ~amb_choice & ~amb_region)):
            res.reasons[name] = res.reasons.get(name, 0) + int((m & ~excluded[idx]).sum())
        excluded[idx[amb_choice | amb_region | amb_cut]] = True
        if mutant == "is_inside":  # pushes the points below the surface out along the normal, as the other shapes do
            inside = surface_below(fld, l) & (depth > rc.EPS32)
            nrm = d / np.where(depth > 0, depth, 1.0)[:, None]
            ii = idx[inside]
            res.pos[ii] = p[ii] - nrm[inside] * (depth[inside] + 0.1 * float(F(r)))[:, None]
        emit = ~beyond
        at, e_at = (q, eq[:, None] * np.ones(3)) if mutant == "local_point_velocity" else (qw, e_qw)
        sv, esv = rc.body_velocity(at, e_at, col)
        keep = emit | excluded[idx]
        sidx = np.concatenate([idx[keep], amb_extra])
        nanx = np.full((len(amb_extra), 3), np.nan)
        S = dict(idx=sidx, q=np.concatenate([qw[keep], nanx]), eq=np.concatenate([e_qw[keep], nanx]), v=np.concatenate([sv[keep], nanx]),
                 ev=np.concatenate([esv[keep], nanx]), amb=np.concatenate([excluded[idx][keep], np.ones(len(amb_extra), bool)]))
        o = np.argsort(S["idx"], kind="stable")
        samples[k] = {key: val[o] for key, val in S.items()}
    res.samples = samples
    res.excluded = excluded | res.excluded
    return res


def query64(fld, pts, R, t, radius, e_pts=0.0):
    """particles_intersecting_shape's decision for a heightfield: distance_to_point(pos, p, solid) <= radius, the unsigned
    distance to the closest point (is_inside is always false).  Returns (hit, decided): `decided` is False where the float32
    distance may lie on either side of the radius (the band)."""
    P = rc._f64(pts)
    R = rc._f64(R).reshape(3, 3)
    t = rc._f64(t)
    l = (P - t) @ R
    el = e_pts + 8 * G * U * (np.abs(P).max(axis=1) + np.abs(t).max())
    _, _, D, eD, _, amb_choice, _ = project64(fld, l, el)
    radius = float(F(radius))
    return D <= radius, ~rc._near(D - radius, eD + 2 * U * radius) & ~(amb_choice & rc._near(D - radius, 4 * eD + 2 * U * radius))
