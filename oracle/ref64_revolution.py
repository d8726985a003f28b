"""Float64 restatement of parry's Cylinder and Cone (axis along local y; half height a, radius r; the cone's apex at (0, a, 0)
and its base disc at y = -a) as the project's contract states them (DESIGN.md sections 10 and 11): ray sampling, contact
sampling and particles_intersecting_shape, each output with a bound on the device's float32 evaluation.

TEST INFRASTRUCTURE ONLY.  Written from the contract, not from salva_b200/contact_sampling.py (the float32 restatement the
device is held to bit for bit): that one is checked against this one.  It extends oracle/ref64_sampling.py (whose traversal
runs unchanged, with this module's AABB and crossings) and reuses the helpers and candidate rules of oracle/ref64_colliders.py.

Crossings.  Exact in float64 from the float32 ray coordinates, with the bound of the device's float32 evaluation: the disc
test c^2 <= r^2 (grazing within 4 u (r^2 + c^2): the ray is undecided), the cylinder's caps +-a (exact), the cone's slant
a - 2a rho / r (5 u 2a f + 2 u |y|) and the horizontal half chords sqrt(R^2 - c^2) with R = r (a - y) / (2a) (3 u R).

Projection.  In the meridian half-plane (rho, y).  Outside, the closest point of the closed section: a 1-Lipschitz map, so
its bound is the local point's bound plus the rounding of its formula.  Inside (surface included), the foot on the nearest
edge: side / slant first, then bottom, then top.  The lift back along u = (x, z) / rho turns a bound e on the point into
qr e / rho on the foot.

Exclusions (counted per reason).  inside: an inside test (rho against r, |y| against a, the slant) within its bound;
edge_tie: two edge distances within their bounds; axis: a foot lifted from a rho within its bound of 0; depth_cut: depth
within its bound of 1.5 h; cell_or_aabb: the candidate gates, as ref64_colliders.  For a query the band is the distance
within its bound of the radius, with the cell box's keys decided as ref64_colliders decides them.

`mutant=` (contact and query) and `bugs=` (sampling) apply one plausible bug to the reference: a bound that passes it is too
loose.
"""
import math
import types

import numpy as np

from oracle import ref64_colliders as rc
from oracle import ref64_sampling as rs

F = np.float32
U = rc.U
G = rc.G
CAPSULE, CYLINDER, CONE = 3, 5, 6
SAMPLE_BUGS = ("apex_at_minus_a",  # the cone's apex at -a and its base at +a
               "axis_along_z",     # the axis along local z
               "radius_at_apex",   # the cone's horizontal radius r (a + y) / (2a): the full radius at the apex end
               "open_caps",        # the cylinder's caps are not hit: vertical rays miss
               "rho2")             # the cone's vertical crossing at a - 2a rho^2 / r^2
CONTACT_MUTANTS = ("apex_at_minus_a", "axis_along_z", "local_point_velocity")
QUERY_MUTANTS = ("abs_r_box", "cone_box_centred", "apex_at_minus_a")


# -- ray sampling ------------------------------------------------------------------------------------------------------------
def aabb(shape):
    """compute_aabb(&Isometry::identity()): [-r, -a, -r] to [r, a, r], exact in float32."""
    if shape.kind not in (CYLINDER, CONE):
        return rs.aabb(shape)
    a, r = shape.params[0], shape.params[1]
    z = F(0)
    return np.array([z - r, -a, z - r], F), np.array([z + r, a, z + r], F)


def crossings(shape, hf, i, cj, ck, bugs=()):
    """ref64_sampling.crossings for cylinders and cones: ascending (X, eX) and the position from which the ray is undecided."""
    if shape.kind not in (CYLINDER, CONE):
        return rs.crossings(shape, hf, i, cj, ck)
    a, r = float(shape.params[0]), float(shape.params[1])
    ax = 2 if "axis_along_z" in bugs else 1
    c = [0.0, 0.0, 0.0]
    c[(i + 1) % 3], c[(i + 2) % 3] = float(cj), float(ck)
    if i == ax:  # along the axis, at rho^2 = c2
        c2 = sum(c[b] * c[b] for b in range(3) if b != ax)
        S, eS = r * r - c2, 4 * U * (r * r + c2)
        if S < -eS:
            return [], math.inf
        if abs(S) <= eS:
            return [], -math.inf
        if shape.kind == CYLINDER:
            return ([] if "open_caps" in bugs else [(-a, 0.0), (a, 0.0)]), math.inf
        f = 0.0 if c2 == 0 else (c2 / (r * r) if "rho2" in bugs else math.sqrt(c2) / r)
        top = a - 2 * a * f
        e = G * (5 * U * 2 * a * f + 2 * U * abs(top))
        if "apex_at_minus_a" in bugs:
            return [(-top, e), (a, 0.0)], math.inf
        return [(-a, 0.0), (top, e)], math.inf
    y = c[ax]
    cc = [c[b] for b in range(3) if b != ax and b != i][0]
    if abs(y) > a:
        return [], math.inf
    if shape.kind == CYLINDER:
        return rs._sqrt_pair(r * r - cc * cc, 4 * U * (r * r + cc * cc))
    if a == 0:
        R = r
    else:
        R = r * ((a + y) if ("apex_at_minus_a" in bugs or "radius_at_apex" in bugs) else (a - y)) / (2 * a)
    return rs._sqrt_pair(R * R - cc * cc, 10 * U * (R * R + cc * cc))


def sample(shape, particle_rad, volume, bugs=()):
    """ref64_sampling.sample with this module's AABB and crossings: the traversal's code runs unchanged, rebound to them."""
    g = dict(vars(rs))
    g["aabb"] = aabb
    g["crossings"] = lambda s, hf, i, cj, ck: crossings(s, hf, i, cj, ck, bugs)
    g["grid"] = types.FunctionType(rs.grid.__code__, g)
    return types.FunctionType(rs.sample.__code__, g)(shape, particle_rad, volume, bugs)


# -- projection --------------------------------------------------------------------------------------------------------------
def _near(x, tol):
    return np.abs(x) <= tol


def project64(kind, a, r, l, nel, mutant=None):
    """The non-solid projection of local points l (m, 3) float64 whose float32 evaluation lies within nel (m,) of them.
    Returns dict(q, eq (m,), inside, D (solid distance), eD, amb_inside, amb_tie, amb_axis)."""
    a, r = float(a), float(r)
    l = np.array(l, np.float64)
    if mutant == "axis_along_z":
        l = l[:, [0, 2, 1]]
    if mutant == "apex_at_minus_a" and kind == CONE:
        l[:, 1] = -l[:, 1]
    m = len(l)
    lx, y, lz = l[:, 0], l[:, 1], l[:, 2]
    rho = np.hypot(lx, lz)
    e_rho = G * nel + 3 * U * rho
    e_y = G * nel
    rnd = 8 * U * (a + r + np.abs(y) + rho)  # the rounding of each formula's handful of operations
    qr, qy = np.zeros(m), np.zeros(m)
    keep = np.zeros(m, bool)
    if kind == CYLINDER:
        inside = (rho <= r) & (np.abs(y) <= a)
        sure_out = (rho > r + e_rho) | (np.abs(y) > a + e_y)
        amb_in = ~sure_out & (_near(rho - r, e_rho) | _near(np.abs(y) - a, e_y))
        ds, db, dt = r - rho, y + a, a - y
        side = (ds <= db) & (ds <= dt)
        bot = ~side & (db <= dt)
        srt = np.sort(np.stack([ds, db, dt], axis=1), axis=1)
        amb_tie = inside & _near(srt[:, 1] - srt[:, 0], e_rho + e_y + 2 * U * (a + r + np.abs(y)))
        keep = np.where(inside, ~side, rho <= r)
        qr = np.where(keep, rho, r)
        qy = np.where(inside, np.where(side, y, np.where(bot, -a, a)), np.clip(y, -a, a))
    else:
        a2, L2 = 2 * a, r * r + 4 * a * a
        L = math.sqrt(L2)
        num = r * (a - y) - a2 * rho
        e_num = r * e_y + a2 * e_rho + 4 * U * (r * np.abs(a - y) + a2 * rho)
        inside = (y >= -a) & (y <= a) & (rho <= r) & (num >= 0)
        sure_out = (y < -a - e_y) | (y > a + e_y) | (rho > r + e_rho) | (num < -e_num)
        amb_in = ~sure_out & (_near(y + a, e_y) | _near(y - a, e_y) | _near(rho - r, e_rho) | _near(num, e_num))
        with np.errstate(divide="ignore", invalid="ignore"):
            dsl = num / L if L > 0 else np.full(m, np.inf)
            slant = dsl <= y + a
            amb_tie = inside & (L > 0) & _near(dsl - (y + a), e_num / max(L, 1e-300) + e_y + 4 * U * (np.abs(dsl) + a + np.abs(y)))
            w = num / L2 if L2 > 0 else np.zeros(m)
            under = (y < -a) & (rho <= r)
            s = np.clip((r * rho + a2 * (a - y)) / L2, 0, 1) if L2 > 0 else np.zeros(m)
        keep = np.where(inside, ~slant, under)
        qr = np.where(inside, np.where(slant, rho + w * a2, rho), np.where(under, rho, s * r))
        qy = np.where(inside, np.where(slant, y + w * r, -a), np.where(under, -a, a - s * a2))
    # the foot's bound in the meridian plane: 1-Lipschitz outside; inside, the edge foot moves with the point
    e_mer = 2 * G * (e_rho + e_y) + rnd
    lift = ~keep & (qr > 0)
    axis = lift & (rho <= 4 * e_rho)
    exact_axis = rho == 0
    rs_ = np.where(rho > 0, rho, 1.0)
    ux, uz = np.where(exact_axis, 1.0, lx / rs_), np.where(exact_axis, 0.0, lz / rs_)
    q = np.stack([np.where(keep, lx, qr * ux), qy, np.where(keep, lz, qr * uz)], axis=1)
    eq = e_mer + np.where(lift & ~exact_axis, 2 * qr * e_rho / rs_, 0.0) + np.where(keep, G * nel, 0.0)
    D = np.where(inside, 0.0, np.hypot(rho - qr, y - qy))
    eD = 2 * G * (e_rho + e_y) + rnd
    if mutant == "apex_at_minus_a" and kind == CONE:
        q[:, 1] = -q[:, 1]
    if mutant == "axis_along_z":
        q = q[:, [0, 2, 1]]
    return dict(q=q, eq=eq, inside=inside, D=D, eD=eD, amb_inside=amb_in, amb_tie=amb_tie, amb_axis=axis & ~exact_axis)


def _capsule64(a, r, l, nel):
    """ref64_colliders' capsule projection and its bounds, in this module's form."""
    cy = np.clip(l[:, 1], -a, a)
    dvec = np.stack([l[:, 0], l[:, 1] - cy, l[:, 2]], axis=1)
    dn = np.linalg.norm(dvec, axis=1)
    axis_ = dn == 0
    dns = np.where(axis_, 1.0, dn)
    s = r / dns
    q = np.stack([np.where(axis_, r, l[:, 0] * s), np.where(axis_, cy, cy + dvec[:, 1] * s), np.where(axis_, 0.0, l[:, 2] * s)], axis=1)
    eq = 2 * G * r * nel / dns + 5 * G * U * r + nel + G * U * (np.abs(cy) + r)
    eq = np.where(axis_, nel, eq)
    amb_in = rc._near(dn - r, G * (nel + 3 * U * np.maximum(dn, r)))
    amb_geo = (~axis_ & (dn <= G * nel)) | rc._near(np.abs(l[:, 1]) - a, nel)
    return dict(q=q, eq=eq, inside=dn <= r, amb_inside=amb_in, amb_tie=np.zeros(len(l), bool), amb_axis=amb_geo)


def posed_box64(kind, a, r, R, t, mutant=None):
    """compute_aabb(pos): the tight support-map box of a cylinder or cone (mins, maxs) and its float32 bound."""
    a, r = float(a), float(r)
    s = np.hypot(R[:, 0], R[:, 2])
    ay = a * R[:, 1]
    if mutant == "abs_r_box":  # |R| e of the local box
        ext = np.abs(R) @ np.array([r, a, r])
        lo, hi = t - ext, t + ext
    elif kind == CYLINDER:
        ext = a * np.abs(R[:, 1]) + r * s
        lo, hi = t - ext, t + ext
    else:
        lo, hi = t + np.minimum(ay, -ay - r * s), t + np.maximum(ay, -ay + r * s)
        if mutant == "cone_box_centred":
            ext = (hi - lo) / 2
            lo, hi = t - ext, t + ext
    e = G * U * (6 * (a + r) + 2 * (np.abs(t) + np.abs(lo) + np.abs(hi)))
    return lo, hi, e


def contact64(pos, vel, colliders, dt, h, radius, mutant=None):
    """update_boundaries over capsule, cylinder and cone colliders in slot order (dicts as ref64_colliders.contact64), with
    the running state and its bound carried from collider to collider.  Returns a ref64_colliders.Contact."""
    P0 = rc._f64(pos)
    N = len(P0)
    p, v = P0.copy(), rc._f64(vel)
    ep, ev = np.zeros((N, 3)), np.zeros((N, 3))
    excluded = np.zeros(N, bool)
    hh = float(F(h))
    cut = 1.5 * hh
    margin = 0.1 * float(F(radius))
    dtp = float(F(dt))
    c_lo, c_hi = rc._cell_range(P0, hh)
    res = rc.Contact()
    res.samples, res.reasons, res.candidates = [None] * len(colliders), {}, 0
    in_cell = np.floor(P0 / hh)

    def exclude(mask, idx, reason):
        n = int((mask & ~excluded[idx]).sum())
        if n:
            res.reasons[reason] = res.reasons.get(reason, 0) + n
        excluded[idx[mask]] = True

    for k, col in enumerate(colliders):
        kind = col["kind"]
        a, r = (float(F(x)) for x in col["params"][:2])
        R = rc._f64(col.get("rotation", np.eye(3))).reshape(3, 3)
        t = rc._f64(col.get("translation", (0, 0, 0)))
        perm = rc._signed_perm(R)
        if kind == CAPSULE:
            ext = rc.posed_ext(col)
            lo, hi, e_box = t - ext, t + ext, G * U * (3 * ext + 2 * (np.abs(t) + ext))
        else:
            lo, hi, e_box = posed_box64(kind, a, r, R, t, mutant)
        mins, maxs = lo - cut, hi + cut
        e_box = e_box + G * U * (np.abs(mins) + np.abs(maxs) + cut)
        lo_q, hi_q = mins / hh, maxs / hh
        lo_tol, hi_tol = e_box / hh + G * U * np.abs(lo_q), e_box / hh + G * U * np.abs(hi_q)
        klo = (np.floor(lo_q - lo_tol), np.floor(lo_q + lo_tol))
        khi = (np.floor(hi_q - hi_tol), np.floor(hi_q + hi_tol))
        sure_in = np.all((c_lo >= klo[1]) & (c_hi <= khi[0]), axis=1)
        sure_out = np.any((c_hi < klo[0]) | (c_lo > khi[1]), axis=1)
        in_box = np.all((in_cell >= np.floor(lo_q)) & (in_cell <= np.floor(hi_q)), axis=1)
        pr_all = p + v * dtp
        known = np.all((ep == 0) & (ev == 0), axis=1)
        f32 = (p.astype(F) + v.astype(F) * F(dtp)).astype(np.float64)
        e_gen = ep + ev * dtp + G * U * (2 * np.abs(v) * dtp + np.abs(p))
        e_pr_all = np.where(known[:, None], np.abs(f32 - pr_all), e_gen)
        s_box = np.minimum(pr_all - mins, maxs - pr_all)
        tol_box = e_pr_all + e_box
        aabb = np.all(s_box >= 0, axis=1)
        maybe = ~sure_out & ~np.any(s_box < -tol_box, axis=1)
        exclude((~sure_in | ~np.all(s_box > tol_box, axis=1)) & maybe, np.arange(N), "cell_or_aabb")
        res.candidates += int(in_box.sum())
        idx = np.nonzero(in_box & aabb)[0]
        amb_extra = np.nonzero(~sure_out & excluded & ~(in_box & aabb))[0]
        pr, e_pr = pr_all[idx], e_pr_all[idx]
        pi, vi, epi, evi = p[idx], v[idx], ep[idx], ev[idx]
        w = pr - t
        e_w = rc._rn(w, e_pr)
        l = w @ R
        e_l = e_w @ np.abs(R)
        if not perm:
            e_l = e_l + G * 3 * U * (np.abs(w) @ np.abs(R))
        nel = np.linalg.norm(e_l, axis=1)
        P = _capsule64(a, r, l, nel) if kind == CAPSULE else project64(kind, a, r, l, nel, mutant)
        q, inside = P["q"], P["inside"]
        qw = q @ R.T + t
        e_qw = P["eq"][:, None] + G * U * np.abs(qw)
        if not perm:
            e_qw = e_qw + G * 3 * U * (np.abs(q) @ np.abs(R).T)
        d = pr - qw
        e_d = e_pr + e_qw + G * U * np.abs(d)
        ned = np.linalg.norm(e_d, axis=1)
        depth = np.linalg.norm(d, axis=1)
        e_depth = G * (ned + 2.5 * U * depth)
        has_n = depth > rc.EPS32
        amb_eps = rc._near(depth - rc.EPS32, e_depth)
        deps = np.where(depth > 0, depth, 1.0)
        n = d / deps[:, None]
        e_n = (2 * G * ned / deps)[:, None] + 3 * G * U
        push = has_n & inside
        ve = np.sum(n * vi, axis=1)
        e_ve = np.sum(np.abs(vi) * e_n + np.abs(n) * evi, axis=1) + 3 * G * U * np.sum(np.abs(n * vi), axis=1)
        beyond = has_n & ~inside & (depth > cut)
        amb_cut = (has_n | amb_eps) & ~inside & rc._near(depth - cut, e_depth + U * cut)
        for name, msk in (("inside", P["amb_inside"]), ("edge_tie", P["amb_tie"]), ("axis", P["amb_axis"]),
                          ("depth_cut", amb_cut), ("normal", (amb_eps & (inside | P["amb_inside"])) | (push & rc._near(ve, e_ve)))):
            exclude(msk, idx, name)
        sdep = depth + margin
        e_s = e_depth + G * U * sdep + 2 * U * margin
        newp = pi - n * sdep[:, None]
        e_newp = epi + e_n * sdep[:, None] + np.abs(n) * e_s[:, None] + G * U * (np.abs(n) * sdep[:, None] + np.abs(newp))
        dv = push & (ve > 0)
        newv = np.where(dv[:, None], vi - n * ve[:, None], vi)
        e_newv = np.where(dv[:, None], evi + e_n * np.abs(ve)[:, None] + np.abs(n) * e_ve[:, None]
                          + G * U * (np.abs(n * ve[:, None]) + np.abs(newv)), evi)
        p[idx[push]], ep[idx[push]] = newp[push], e_newp[push]
        v[idx[push]], ev[idx[push]] = newv[push], e_newv[push]
        emit = ~beyond
        at, e_at = (q, P["eq"][:, None] * np.ones(3)) if mutant == "local_point_velocity" else (qw, e_qw)
        sv, esv = rc.body_velocity(at, e_at, col)
        keep = emit | excluded[idx]
        nanx = np.full((len(amb_extra), 3), np.nan)
        S = dict(idx=np.concatenate([idx[keep], amb_extra]), q=np.concatenate([qw[keep], nanx]), eq=np.concatenate([e_qw[keep], nanx]),
                 v=np.concatenate([sv[keep], nanx]), ev=np.concatenate([esv[keep], nanx]),
                 amb=np.concatenate([excluded[idx][keep], np.ones(len(amb_extra), bool)]))
        o = np.argsort(S["idx"], kind="stable")
        res.samples[k] = {key: val[o] for key, val in S.items()}
    res.pos, res.vel, res.ep, res.ev, res.excluded = p, v, ep, ev, excluded
    return res


def query64(kind, a, r, pts, R, t, h, radius, mutant=None):
    """particles_intersecting_shape for a cylinder or cone: a point is reported when its cell lies in the keys of the posed
    box and distance_to_point(solid) <= radius.  Returns (hit, decided) per point; `decided` is False in the band where a key
    or the distance lies within its bound of the decision."""
    P = rc._f64(pts)
    R = rc._f64(R).reshape(3, 3)
    t = rc._f64(t)
    hh = float(F(h))
    lo, hi, e_box = posed_box64(kind, a, r, R, t, mutant)
    lo_q, hi_q = lo / hh, hi / hh
    tl, th = e_box / hh + G * U * np.abs(lo_q), e_box / hh + G * U * np.abs(hi_q)
    c_lo, c_hi = rc._cell_range(P, hh)
    cells_in = np.all((c_lo >= np.floor(lo_q + tl)) & (c_hi <= np.floor(hi_q - th)), axis=1)
    cells_out = np.any((c_hi < np.floor(lo_q - tl)) | (c_lo > np.floor(hi_q + th)), axis=1)
    in_cells = np.all((np.floor(P / hh) >= np.floor(lo_q)) & (np.floor(P / hh) <= np.floor(hi_q)), axis=1)
    l = (P - t) @ R
    nel = 8 * G * U * (np.abs(P).max(axis=1) + np.abs(t).max())
    pr = project64(kind, a, r, l, nel, mutant if mutant == "apex_at_minus_a" else None)
    radius = float(F(radius))
    D, eD = pr["D"], pr["eD"] + 2 * U * radius
    hit = in_cells & (D <= radius)
    decided = (cells_in | cells_out) & ~(rc._near(D - radius, eD) & ~cells_out)
    return hit, decided


# ---- scenes: shared by the CPU checks of the float32 restatement and the GPU checks of the device ------------------------
def _posed():
    """Slot order: a rotated dynamic cylinder, a rotated dynamic cone overlapping the rotated dynamic capsule of the next
    slot, a fixed cone and a parentless cylinder with signed-permutation rotations; two fluids with different groups, and
    particles at rest on the exact axes of the last two."""
    R = 0.05
    rng = np.random.default_rng(13)
    a = rc.lattice((9, 8, 9), R * 1.9, (0.05, 0.08, 0.05), seed=13, amplitude=0.2)
    va = rng.normal(0, 3.0, a.shape).astype(F)
    b = (rng.random((300, 3)) * np.array([0.8, 0.7, 0.8]) + np.array([0.0, 0.05, 0.0])).astype(F)
    vb = rng.normal(0, 2.0, b.shape).astype(F)

    def states(k):
        return [rc._state((0.3, 0.3 - k / 256.0, 0.3), rc.rot(0.3 + 0.1 * k, 0.2, 0.5), rc.BODY_DYNAMIC, (0, -1, 0), (0.5, 2, -1)),
                rc._state((0.5, 0.35, 0.45), rc.rot(0.7, -0.4 + 0.05 * k, 0.9), rc.BODY_DYNAMIC, (0.3, 0, 0.1), (0, 1.5, 2), (0.45, 0.3, 0.45)),
                rc._state((0.55, 0.42, 0.5), rc.rot(0.2, 0.9, -0.3), rc.BODY_DYNAMIC, (0, 0, 0), (-1, 0, 3)),
                rc._state((0.25, 0.625, 0.625), rc.RZ90, rc.BODY_FIXED, (0.25, 0, 0), (0, 0, 1)),
                rc._state((0.75, 0.25, 0.25), rc.RX90, rc.BODY_NONE, (1, 1, 1), (1, 1, 1))]
    shapes = [(CYLINDER, (0.12, 0.1)), (CONE, (0.15, 0.12)), (CAPSULE, (0.1, 0.06)), (CONE, (0.125, 0.125)), (CYLINDER, (0.0625, 0.125))]
    st = states(0)
    ex = np.asarray([s["rotation"] @ np.asarray(l, F) + s["translation"] for s, l in
                     ((st[3], (0, -0.03125, 0)), (st[3], (0, 0.0625, 0)), (st[4], (0, 0, 0)), (st[4], (0, 0.03125, 0)))], F)
    b = np.concatenate([b, ex])
    vb = np.concatenate([vb, np.zeros_like(ex)])
    return dict(radius=R, fluids=[dict(positions=a, velocities=va, memberships=1, filter=1), dict(positions=b, velocities=vb)],
                shapes=shapes, boundary_of_slot=[3, 5, 1, 2, 4], plain=True, states=states, steps=6)


def _degenerate():
    """A disc (zero-height cylinder), a segment (zero-radius cylinder), a flat cone and a needle cone in one fluid block."""
    R = 0.05
    a = rc.lattice((8, 6, 8), R * 1.9, (0.0, 0.0, 0.0), seed=17, amplitude=0.2)
    va = np.random.default_rng(17).normal(0, 1.0, a.shape).astype(F)

    def states(k):
        return [rc._state((0.2, 0.3, 0.2), rc.rot(0.3, 0.1 * k, 0.2), rc.BODY_DYNAMIC, (0, 1, 0), (1, 0, 0)),
                rc._state((0.55, 0.3, 0.2), rc.rot(0.5, 0.2, 0.1), rc.BODY_DYNAMIC, (0, 0, 1), (0, 2, 0)),
                rc._state((0.2, 0.3, 0.55), None, rc.BODY_FIXED),
                rc._state((0.55, 0.3, 0.55), rc.rot(0.1, 0.4, 0.2 + 0.1 * k), rc.BODY_DYNAMIC, (0.5, 0, 0), (0, 0, 1))]
    return dict(radius=R, fluids=[dict(positions=a, velocities=va)],
                shapes=[(CYLINDER, (0.0, 0.12)), (CYLINDER, (0.15, 0.0)), (CONE, (0.0, 0.12)), (CONE, (0.15, 0.0))],
                boundary_of_slot=[0, 1, 2, 3], plain=False, states=states, steps=4)


SCENES = dict(posed=_posed, degenerate=_degenerate)
