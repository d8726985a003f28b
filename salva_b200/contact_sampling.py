"""DynamicContactSampling (fluids_pipeline.rs:192-255) restated in numpy float32.

Every operation below is one float32 operation in the order k_contact_sample (csrc/sph_shapes.cuh) performs it, so the
restatement is bit-identical to the device path.  ContactSamplingHook runs it as a host CouplingManager, through
LiquidWorld.step_with_coupling: the way to contact-sample without the device path, and the yardstick the device path is
checked and timed against.
"""
import numpy as np

from .liquid_world import BODY_NONE, CouplingManager

F32 = np.float32
EPS = F32(np.finfo(np.float32).eps)  # Unit::try_new_and_get(dpt, f32::EPSILON)
BALL, CUBOID, CAPSULE, HEIGHTFIELD, CYLINDER, CONE = 1, 2, 3, 4, 5, 6
NO_TRI = 2 ** 32 - 1  # no triangle yet (the device's UINT32_MAX)


def _dot(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def hf_grid(heights, scale):
    """The host constants of a heightfield (csrc/sph_colliders_host.inl hf_check): half extents, cell sizes, height scale, the scaled
    height range."""
    H = np.ascontiguousarray(heights, F32)
    sx, sy, sz = (F32(x) for x in scale)
    nr, nc = H.shape
    g = dict(H=H, nrows=nr, ncols=nc, hx=sx * F32(0.5), hz=sz * F32(0.5), sy=sy, dx=sx / F32(nc - 1), dz=sz / F32(nr - 1))
    g["dmin"] = min(g["dx"], g["dz"])
    g["ylo"], g["yhi"] = H.min() * sy, H.max() * sy
    return g


def hf_margin(g, cap):
    """The search margin M = 2^-10 (sx/2 + sz/2 + max |y| + cap) of hf_set_cap."""
    return (((g["hx"] + g["hz"]) + max(abs(g["ylo"]), abs(g["yhi"]))) + F32(cap)) * F32(2.0 ** -10)


def posed_aabb(kind, params, rotation, translation, hf=None):
    """The posed shape's AABB (shape.compute_aabb(pos)): translation -/+ the half extents sph_world_particles_in_shape uses;
    for a heightfield (hf: hf_grid) Aabb::transform_by of its local box, centre R c + t and half extents |R| e."""
    if kind == HEIGHTFIELD:
        R = np.asarray(rotation, F32).reshape(3, 3)
        t = np.asarray(translation, F32)
        cy, ey = (hf["ylo"] + hf["yhi"]) * F32(0.5), (hf["yhi"] - hf["ylo"]) * F32(0.5)
        ext = np.array([(abs(R[a, 0]) * hf["hx"] + abs(R[a, 1]) * ey) + abs(R[a, 2]) * hf["hz"] for a in range(3)], F32)
        c = np.array([R[a, 1] * cy + t[a] for a in range(3)], F32)
        return c - ext, c + ext
    R = np.asarray(rotation, F32).reshape(3, 3)
    p = np.zeros(4, F32)
    p[:len(params)] = np.asarray(params, F32)
    t = np.asarray(translation, F32)
    if kind in (CYLINDER, CONE):  # parry's tight support-map box
        mins, maxs = np.empty(3, F32), np.empty(3, F32)
        a, r = p[0], p[1]
        for i in range(3):
            si = np.sqrt(R[i, 0] * R[i, 0] + R[i, 2] * R[i, 2])
            ay, rs = a * R[i, 1], r * si
            if kind == CYLINDER:
                ext = abs(R[i, 1]) * a + rs
                mins[i], maxs[i] = t[i] - ext, t[i] + ext
            else:
                mins[i], maxs[i] = t[i] + min(ay, -ay - rs), t[i] + max(ay, -ay + rs)
        return mins, maxs
    ext = np.empty(3, F32)
    for a in range(3):
        if kind == BALL:
            ext[a] = p[0]
        elif kind == CUBOID:
            ext[a] = (abs(R[a, 0]) * p[0] + abs(R[a, 1]) * p[1]) + abs(R[a, 2]) * p[2]
        else:
            ext[a] = abs(R[a, 1]) * p[0] + p[1]
    return t - ext, t + ext


def _grid(j, last, half, d):
    """smp_grid: vertex coordinate j of a grid of `last` cells of size d from -half (the last one exactly +half)."""
    return np.where(j == last, half, -half + j.astype(F32) * d).astype(F32)


def _cell(c, half, d, cells):
    """smp_cell: the cell of coordinate c, clamped to the grid."""
    t = (c + half) / d
    return np.clip(np.floor(t), 0, cells - 1).astype(np.int64)


def _dot3(a, b):
    return _dot(a[..., 0], a[..., 1], a[..., 2], b[..., 0], b[..., 1], b[..., 2])


def hf_tri(p, a, b, c):
    """hf_tri: the closest point of the closed triangles (a, b, c) to p (Ericson's regions, the device's float32
    operations) and its squared distance; arrays (..., 3)."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
        d1, d2, d3, d4, d5, d6 = _dot3(ab, ap), _dot3(ac, ap), _dot3(ab, bp), _dot3(ac, bp), _dot3(ab, cp), _dot3(ac, cp)
        vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
        e43, e56 = d4 - d3, d5 - d6
        regions = [(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
                   (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)]
        den = F32(1) / ((va + vb) + vc)
        face = (a + ab * (vb * den)[..., None]) + ac * (vc * den)[..., None]
        q = np.select([m[..., None] for m in regions],
                      [a, b, a + (d1 / (d1 - d3))[..., None] * ab, c, a + (d2 / (d2 - d6))[..., None] * ac,
                       b + (e43 / (e43 + e56))[..., None] * (c - b)], face).astype(F32)
        e = p - q
        return q, _dot3(e, e)


def _ring_gap(r, g, margin):
    """The least horizontal distance of ring r's cells, less the margin: (r - 1) dmin - M."""
    return F32(r - 1) * g["dmin"] - margin


def _beats(d, t, best, bidx):
    """(d, t) before (best, bidx) in the order (squared distance, parry triangle index)."""
    return (d < best) | ((d == best) & (t < bidx))


def hf_project_local(g, l, cap):
    """hf_closest for local points l (n, 3) float32: the ring search with the device's stop rule (cap: h + prediction for
    contact sampling, particle_radius for queries).  Returns (q (n, 3), squared distance (n,), found (n,))."""
    l = np.asarray(l, F32)
    n = len(l)
    ni, nj = g["nrows"] - 1, g["ncols"] - 1
    ci, cj = _cell(l[:, 2], g["hz"], g["dz"], ni), _cell(l[:, 0], g["hx"], g["dx"], nj)
    rmax = np.maximum(np.maximum(ci, ni - 1 - ci), np.maximum(cj, nj - 1 - cj))
    cap2, margin = F32(cap) * F32(cap), hf_margin(g, cap)
    best = np.full(n, np.inf, F32)
    bidx = np.full(n, NO_TRI, np.int64)
    q = np.zeros((n, 3), F32)
    active = np.ones(n, bool)
    H, sy = g["H"], g["sy"]
    for r in range(int(rmax.max(initial=0)) + 1):
        active &= r <= rmax
        gap = _ring_gap(r, g, margin)
        if gap > 0:
            active &= ~(gap * gap > np.minimum(best, cap2))
        idx = np.nonzero(active)[0]
        if not len(idx):
            break
        if r == 0:
            di, dj = np.zeros(1, np.int64), np.zeros(1, np.int64)
        else:
            k = np.arange(-r, r + 1)
            m = np.arange(-r + 1, r)
            di = np.concatenate([np.full(2 * r + 1, -r), np.full(2 * r + 1, r), m, m])
            dj = np.concatenate([k, k, np.full(2 * r - 1, -r), np.full(2 * r - 1, r)])
        I, J = ci[idx, None] + di[None, :], cj[idx, None] + dj[None, :]
        ok = (I >= 0) & (I < ni) & (J >= 0) & (J < nj)
        I, J = np.clip(I, 0, ni - 1), np.clip(J, 0, nj - 1)
        x0, x1 = _grid(J, nj, g["hx"], g["dx"]), _grid(J + 1, nj, g["hx"], g["dx"])
        z0, z1 = _grid(I, ni, g["hz"], g["dz"]), _grid(I + 1, ni, g["hz"], g["dz"])
        p00 = np.stack([x0, H[I, J] * sy, z0], -1)
        p10 = np.stack([x1, H[I, J + 1] * sy, z0], -1)
        p01 = np.stack([x0, H[I + 1, J] * sy, z1], -1)
        p11 = np.stack([x1, H[I + 1, J + 1] * sy, z1], -1)
        p = l[idx, None, :]
        qa, da = hf_tri(p, p00, p10, p01)
        qb, db = hf_tri(p, p10, p11, p01)
        base = 2 * (J * ni + I)
        D = np.concatenate([da, db], 1)
        T = np.concatenate([base, base + 1], 1)
        Q = np.concatenate([qa, qb], 1)
        bad = ~np.concatenate([ok, ok], 1) | np.isnan(D)  # NaN never wins on the device
        D = np.where(bad, F32(np.inf), D)
        T = np.where(bad, 2 ** 40, T)
        dm = D.min(axis=1)
        win = np.where(D == dm[:, None], T, 2 ** 41).argmin(axis=1)
        rows = np.arange(len(idx))
        rd, rt = D[rows, win], T[rows, win]
        take = _beats(rd, rt, best[idx], bidx[idx])
        best[idx[take]], bidx[idx[take]] = rd[take], rt[take]
        q[idx[take]] = Q[rows, win][take]
    return q, best, bidx != NO_TRI


def rev_meridian(kind, a, r, rho, y):
    """rev_meridian: the meridian foot (qr, qy) of a cylinder or cone (half height a, radius r) for points (rho, y), whether
    the point is inside (surface included) and whether the foot keeps the point's rho."""
    a, r = F32(a), F32(r)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == CYLINDER:
            inside = (rho <= r) & (np.abs(y) <= a)
            ds, db, dt = r - rho, y + a, a - y
            keep_in = ~((ds <= db) & (ds <= dt))
            qy_in = np.where(~keep_in, y, np.where(db <= dt, -a, a))
            keep = np.where(inside, keep_in, rho <= r)
            qr = np.where(keep, rho, r)
            qy = np.where(inside, qy_in, np.minimum(np.maximum(y, -a), a))
            return qr.astype(F32), qy.astype(F32), inside, keep
        a2 = a + a
        L2 = r * r + a2 * a2
        num = r * (a - y) - a2 * rho
        inside = (y >= -a) & (y <= a) & (rho <= r) & (num >= 0)
        slant = (L2 > 0) & (num / np.sqrt(L2) <= y + a)
        w = num / L2
        under = (y < -a) & (rho <= r)
        s = np.minimum(np.maximum((r * rho + a2 * (a - y)) / L2, F32(0)), F32(1)) if L2 > 0 else np.zeros_like(rho)
        keep = np.where(inside, ~slant, under)
        qr = np.where(inside, np.where(slant, rho + w * a2, rho), np.where(under, rho, s * r))
        qy = np.where(inside, np.where(slant, y + w * r, -a), np.where(under, -a, a - s * a2))
        return qr.astype(F32), qy.astype(F32), inside, keep


def project_local(kind, params, l):
    """project_point_and_get_feature (non-solid) in the shape's local frame, for points l (n, 3) float32.
    Returns (proj (n, 3), inside (n,), valid (n,)); valid is False where the projection is undefined (a ball's centre)."""
    l = np.asarray(l, F32)
    p = np.zeros(4, F32)
    p[:len(params)] = np.asarray(params, F32)
    lx, ly, lz = l[:, 0], l[:, 1], l[:, 2]
    valid = np.ones(len(l), bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind in (CYLINDER, CONE):  # the meridian foot lifted along (x, z) / rho, along local +x at rho = 0
            rho = np.sqrt(lx * lx + lz * lz)
            qr, qy, inside, keep = rev_meridian(kind, p[0], p[1], rho, ly)
            s = qr / rho
            axis = rho == 0
            q = np.stack([np.where(keep, lx, np.where(axis, qr, lx * s)), qy, np.where(keep, lz, np.where(axis, F32(0), lz * s))], axis=1)
        elif kind == BALL:
            n2 = _dot(lx, ly, lz, lx, ly, lz)
            valid = n2 != 0
            inside = n2 <= p[0] * p[0]
            s = p[0] / np.sqrt(n2)
            q = np.stack([lx * s, ly * s, lz * s], axis=1)
        elif kind == CUBOID:
            mp = -p[:3] - l
            pm = l - p[:3]
            sh = np.maximum(mp, F32(0)) - np.maximum(pm, F32(0))
            inside = np.all(sh == 0, axis=1)
            best = np.full(len(l), -np.finfo(np.float32).max, F32)
            bid = np.zeros(len(l), np.int64)
            is_mins = np.zeros(len(l), bool)
            for a in range(3):  # nearest face: a tie goes to the mins face, a tie across axes keeps the lowest axis
                c1 = mp[:, a] < pm[:, a]
                tmax = c1 & (pm[:, a] > best)
                tmin = ~c1 & (mp[:, a] > best)
                bid = np.where(tmax | tmin, a, bid)
                is_mins = np.where(tmax, False, np.where(tmin, True, is_mins))
                best = np.where(tmax, pm[:, a], np.where(tmin, mp[:, a], best))
            shin = np.zeros_like(l)
            shin[np.arange(len(l)), bid] = np.where(is_mins, best, -best)
            sh = np.where(inside[:, None], shin, sh)
            q = l + sh
        else:
            cy = np.minimum(np.maximum(ly, -p[0]), p[0])
            dy = ly - cy
            dn = np.sqrt(_dot(lx, dy, lz, lx, dy, lz))
            inside = dn <= p[1]
            s = p[1] / dn
            axis = dn == 0  # on the segment: along local +x
            q = np.stack([np.where(axis, p[1], lx * s), np.where(axis, cy, cy + dy * s), np.where(axis, F32(0), lz * s)], axis=1)
    return q.astype(F32), inside, valid


def velocity_at(points, body, linvel, angvel, world_com):
    """body.velocity_at_point(p) at the WORLD points, zero without a parent body."""
    if body == BODY_NONE:
        return np.zeros_like(points)
    lv, w, c = (np.asarray(x, F32) for x in (linvel, angvel, world_com))
    d = points - c
    return np.stack([lv[0] + (w[1] * d[:, 2] - w[2] * d[:, 1]),
                     lv[1] + (w[2] * d[:, 0] - w[0] * d[:, 2]),
                     lv[2] + (w[0] * d[:, 1] - w[1] * d[:, 0])], axis=1).astype(F32)


def contact_sample(pos, vel, colliders, dt, h, particle_radius, branches=None):
    """One update_boundaries over every fluid particle (pos, vel: (n, 3) float32 in global original order) and the contact
    colliders in slot order, each a dict(kind, params, rotation, translation, body, linvel, angvel, world_com), a heightfield
    (kind 4) with heights (nrows, ncols) and scale instead of params; the pose defaults to the identity, the rest to a
    parentless collider.  `dt` is
    the lagging timestep.  Returns (pos, vel, samples) with the pushes applied and samples[k] = (positions, velocities)
    of collider k in original particle order.  `branches` (a dict) counts, over all colliders, the candidates that took each
    branch of the rule: pushed, shell (outside, kept), beyond (outside by more than h + prediction), on_surface (|dpt| <=
    f32::EPSILON), prediction_outside (cell in the box, prediction outside the AABB), cell_outside (prediction inside the
    AABB, cell outside the box: not a candidate)."""
    pos = np.array(pos, F32, copy=True)
    vel = np.array(vel, F32, copy=True)
    h, dt = F32(h), F32(dt)
    prediction = h * F32(0.5)
    cut = h + prediction
    margin = F32(particle_radius) * F32(0.1)
    cells = np.floor(pos / h)  # the hgrid cells of the positions at the start of the substep
    samples = []
    for col in colliders:
        R = np.asarray(col.get("rotation", np.eye(3)), F32).reshape(3, 3)  # the identity pose by default, as sph_collider_register
        t = np.asarray(col.get("translation", (0.0, 0.0, 0.0)), F32)
        hf = hf_grid(col["heights"], col["scale"]) if col["kind"] == HEIGHTFIELD else None
        mins, maxs = posed_aabb(col["kind"], col.get("params", ()), R, t, hf)
        mins, maxs = mins - cut, maxs + cut
        lo, hi = np.floor(mins / h), np.floor(maxs / h)
        in_box = np.all((cells >= lo) & (cells <= hi), axis=1)
        idx = np.nonzero(in_box)[0]
        p, v = pos[idx], vel[idx]
        pr = p + v * dt
        keep = np.all((pr >= mins) & (pr <= maxs), axis=1)
        if branches is not None:
            pr_all = pos + vel * dt
            out_box = ~in_box & np.all((pr_all >= mins) & (pr_all <= maxs), axis=1)
            branches["prediction_outside"] = branches.get("prediction_outside", 0) + int((~keep).sum())
            branches["cell_outside"] = branches.get("cell_outside", 0) + int(out_box.sum())
        idx, p, v, pr = idx[keep], p[keep], v[keep], pr[keep]
        w = pr - t
        l = np.stack([_dot(R[0, a], R[1, a], R[2, a], w[:, 0], w[:, 1], w[:, 2]) for a in range(3)], axis=1).astype(F32)
        if hf is not None:  # is_inside is always false: no push
            q, _, valid = hf_project_local(hf, l, cut)
            inside = np.zeros(len(l), bool)
        else:
            q, inside, valid = project_local(col["kind"], col["params"], l)
        idx, p, v, pr, q, inside = idx[valid], p[valid], v[valid], pr[valid], q[valid], inside[valid]
        qw = np.stack([_dot(R[a, 0], R[a, 1], R[a, 2], q[:, 0], q[:, 1], q[:, 2]) + t[a] for a in range(3)], axis=1).astype(F32)
        d = pr - qw
        depth = np.sqrt(_dot(d[:, 0], d[:, 1], d[:, 2], d[:, 0], d[:, 1], d[:, 2]))
        has_n = depth > EPS
        with np.errstate(divide="ignore", invalid="ignore"):
            n = d / depth[:, None]
        push = has_n & inside
        s = (depth + margin)[:, None]
        ve = _dot(n[:, 0], n[:, 1], n[:, 2], v[:, 0], v[:, 1], v[:, 2])
        vn = np.where((ve > 0)[:, None], v - n * ve[:, None], v)
        pos[idx[push]] = (p - n * s)[push]
        vel[idx[push]] = vn[push]
        emit = ~(has_n & ~inside & (depth > cut))
        if branches is not None:
            for name, m in (("pushed", push), ("shell", has_n & ~inside & emit), ("beyond", ~emit), ("on_surface", ~has_n)):
                branches[name] = branches.get(name, 0) + int(m.sum())
        qe = qw[emit]
        samples.append((qe, velocity_at(qe, col.get("body", BODY_NONE), col.get("linvel", (0, 0, 0)), col.get("angvel", (0, 0, 0)),
                                        col.get("world_com", (0, 0, 0)))))
    return pos, vel, samples


class ContactSamplingHook(CouplingManager):
    """DynamicContactSampling as a host CouplingManager: reads every fluid, runs contact_sample, writes the pushed fluid back
    and replaces each collider's boundary with its samples.  `fluids`: fluid handles in slot order; `entries`: one
    (boundary handle, collider dict) per collider in slot order; update the dicts' poses between steps."""

    def __init__(self, fluids, entries):
        self.fluids, self.entries = list(fluids), list(entries)

    def update_boundaries(self, world, dt, inv_dt, h, particle_radius):
        parts = [world.read_fluid(f) for f in self.fluids]
        sizes = [len(p) for p, _ in parts]
        pos = np.concatenate([p for p, _ in parts]) if parts else np.zeros((0, 3), F32)
        vel = np.concatenate([v for _, v in parts]) if parts else np.zeros((0, 3), F32)
        pos2, vel2, samples = contact_sample(pos, vel, [c for _, c in self.entries], dt, h, particle_radius)
        o = 0
        for f, n in zip(self.fluids, sizes):
            if n and not (np.array_equal(pos2[o:o + n], pos[o:o + n]) and np.array_equal(vel2[o:o + n], vel[o:o + n])):
                world.write_fluid(f, pos2[o:o + n], vel2[o:o + n])
            o += n
        for (b, _), (sp, sv) in zip(self.entries, samples):
            world.set_boundary_particles(b, sp, sv)
