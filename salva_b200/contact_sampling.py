"""DynamicContactSampling (fluids_pipeline.rs:192-255) restated in numpy float32.

Every operation below is one float32 operation in the order k_contact_sample (csrc/sph_kernels.cuh) performs it, so the
restatement is bit-identical to the device path.  ContactSamplingHook runs it as a host CouplingManager, through
LiquidWorld.step_with_coupling: the way to contact-sample without the device path, and the yardstick the device path is
checked and timed against.
"""
import numpy as np

from .liquid_world import BODY_NONE, CouplingManager

F32 = np.float32
EPS = F32(np.finfo(np.float32).eps)  # Unit::try_new_and_get(dpt, f32::EPSILON)
BALL, CUBOID, CAPSULE = 1, 2, 3


def _dot(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def posed_aabb(kind, params, rotation, translation):
    """The posed shape's AABB (shape.compute_aabb(pos)): translation -/+ the half extents sph_world_particles_in_shape uses."""
    R = np.asarray(rotation, F32).reshape(3, 3)
    p = np.zeros(4, F32)
    p[:len(params)] = np.asarray(params, F32)
    t = np.asarray(translation, F32)
    ext = np.empty(3, F32)
    for a in range(3):
        if kind == BALL:
            ext[a] = p[0]
        elif kind == CUBOID:
            ext[a] = (abs(R[a, 0]) * p[0] + abs(R[a, 1]) * p[1]) + abs(R[a, 2]) * p[2]
        else:
            ext[a] = abs(R[a, 1]) * p[0] + p[1]
    return t - ext, t + ext


def project_local(kind, params, l):
    """project_point_and_get_feature (non-solid) in the shape's local frame, for points l (n, 3) float32.
    Returns (proj (n, 3), inside (n,), valid (n,)); valid is False where the projection is undefined (a ball's centre)."""
    l = np.asarray(l, F32)
    p = np.zeros(4, F32)
    p[:len(params)] = np.asarray(params, F32)
    lx, ly, lz = l[:, 0], l[:, 1], l[:, 2]
    valid = np.ones(len(l), bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kind == BALL:
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
    colliders in slot order, each a dict(kind, params, rotation, translation, body, linvel, angvel, world_com); the
    pose defaults to the identity, the rest to a parentless collider.  `dt` is
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
        mins, maxs = posed_aabb(col["kind"], col["params"], R, t)
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
