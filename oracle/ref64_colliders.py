"""Float64 restatement of the collider coupling (ColliderCouplingManager::{update_boundaries, transmit_forces},
fluids_pipeline.rs:157-287, as DESIGN.md §10 states the device path), each output with a bound on its float32 evaluation.

TEST INFRASTRUCTURE ONLY.  Written from the reference and DESIGN.md §10, not from salva_b200/contact_sampling.py (the float32
restatement the device is held to bit for bit): that one is checked against this one.

Contact sampling (:192-255).  Colliders in slot order; for each one the posed AABB (ball r, cuboid |R| e, capsule |R_y| a + r,
the half extents of DESIGN.md §10) loosened by h + prediction = 1.5 h (:193, :199); the candidates are the particles whose
start-of-substep cell key floor(x / h) lies in [key(mins), key(maxs)] (:201-204, hgrid.rs); a candidate is kept when its
prediction p + v dt (the lagging dt, :208-209, with the running p and v) lies in the AABB (:211); it is projected in the local
frame l = R^T (pr - t) (:212-216; ball, cuboid with ties to the mins face and the lowest axis, capsule along local y); with
|dpt| <= f32::EPSILON nothing more happens (:220-221); inside, it is pushed by depth + 0.1 r (:224-225) and its normal
velocity removed when n.v > 0 (:227-233); outside by more than 1.5 h it is cut (:234-235); the sample is the WORLD projection
with the body's velocity there (:239-246), zero without a parent body.  Deviations of the engine, restated: a ball's centre
gives no sample; a point on a capsule's axis projects along local +x.

Bounds.  Every output carries a per-component bound on |float32 - float64|, built from the kernel's operation sequence:
one rounding (u = 2^-24) per operation, relative to its operands' magnitudes, plus the propagated bounds of the operands;
a product of second-order terms is covered by a factor G = 1.01.  Where the operands of the prediction and of the local
transform are exactly known (a particle not pushed yet, a signed-permutation rotation) the rounding is taken as its exact
value, so exact geometry (points on a face, a ball's centre, a capsule's axis) is decided without an exclusion.  A normal
n = d / |d| carries 2 |e_d| / |d|; a projection onto a ball or a capsule carries 2 r |e_l| / |l|.  The running state carries
its bound from collider to collider.

Exclusions.  A particle is excluded (from that collider on, for the rest of the step) when a float decision lies inside its
bound: its cell key at a cell face, the box keys at theirs, AABB containment, inside / outside, |dpt| against eps, depth against
1.5 h, the sign of n.v, the nearest-face tie of a cuboid, the capsule's clamp at +-a, a ball's centre, a capsule's axis.  Its
samples may be present or absent; `match_samples` walks the device samples and the reference in key order.

Impulses (:263-287): per dynamic collider sum f dt and sum (p - com) x f dt with the step's dt, fed the boundary forces and
positions read back; fixed bodies, parentless colliders, empty and removed boundaries give zero.  The bound follows
k_collider_impulse's reduction: per-block shared-memory atomics over T terms, then global atomics over G blocks, so
(T + G + c) u sum |terms|.

StaticSampling (:180-191): R l + t, with the body's velocity at the LOCAL point (:183).

`mutant=` applies one plausible bug to the reference instead; a bound that passes it is too loose.
"""
import numpy as np

F = np.float32
U = 2.0 ** -24
G = 1.01
EPS32 = float(np.finfo(np.float32).eps)
BALL, CUBOID, CAPSULE = 1, 2, 3
BODY_NONE, BODY_FIXED, BODY_DYNAMIC = 0, 1, 2
BRANCHES = ("pushed", "shell", "beyond", "prediction_outside", "cell_outside", "on_surface", "ball_centre", "capsule_axis")

CONTACT_MUTANTS = ("local_point_velocity", "current_dt", "current_position", "no_margin", "no_cut", "aabb_not_loosened",
                   "unrotated_aabb", "r_for_rt", "reverse_slot_order", "start_state", "ties_to_maxs", "no_vn_gate")
STATIC_MUTANTS = ("world_point_velocity",)
IMPULSE_MUTANTS = ("lagging_dt", "torque_about_translation", "drop_boundary_slot", "fixed_counted")


def _f64(x):
    return np.asarray(x, F).astype(np.float64)


def _signed_perm(R):
    A = np.abs(R)
    return bool(np.all((A == 0) | (A == 1)) and np.all(A.sum(axis=0) == 1) and np.all(A.sum(axis=1) == 1))


def _rn(x, e):
    """Bound after one float32 rounding of x, whose operands carry the propagated bound e: the exact rounding where e = 0."""
    exact = np.abs(x.astype(F).astype(np.float64) - x)
    return np.where(e == 0, exact, e + G * U * np.abs(x))


def _cross(a, b):
    return np.cross(a, b)


def _cross_abs(a, b):
    """|a| x |b| with every difference an addition: the absolute evaluation of a cross product."""
    a, b = np.abs(a), np.abs(b)
    return np.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], axis=-1)


def body_velocity(x, ex, col):
    """velocity_at_point: linvel + angvel x (x - world_com), with its bound; zero without a parent body."""
    if col.get("body", BODY_NONE) == BODY_NONE:
        return np.zeros_like(x), np.zeros_like(x)
    lv, w, c = (_f64(col.get(k, (0, 0, 0))) for k in ("linvel", "angvel", "world_com"))
    d = x - c
    ed = ex + G * U * np.abs(d)
    v = lv + _cross(w, d)
    e = _cross_abs(w, ed) + 2 * G * U * _cross_abs(w, d) + G * U * (np.abs(v) + np.abs(lv))
    return v, e


def posed_ext(col, mutant=None):
    kind, p = col["kind"], np.zeros(3)
    p[:len(col["params"])] = _f64(col["params"])
    R = _f64(col.get("rotation", np.eye(3))).reshape(3, 3)
    if kind == BALL:
        return np.full(3, p[0])
    if kind == CUBOID:
        return p.copy() if mutant == "unrotated_aabb" else np.abs(R) @ p
    if mutant == "unrotated_aabb":
        return np.array([p[1], p[0] + p[1], p[1]])
    return np.abs(R[:, 1]) * p[0] + p[1]


class Contact:
    """The float64 result of one update_boundaries.  pos, vel, ep, ev: per particle (N, 3); excluded: (N,) bool; samples[k]
    of the k-th collider in the order given: dict(idx, q, eq, v, ev, amb) sorted by original index; branches[kind]: counts."""


def _near(x, tol):
    """A decision inside its bound; with a zero bound the float32 operands are exact and so is the decision."""
    return (np.abs(x) <= tol) & (tol > 0)


def _cell_range(x, h):
    """[lo, hi] of floor(fl(x / h)) for float32 x (exact) and h: one rounding, exact where x / h is a float32."""
    q = x / h
    exact = q.astype(F).astype(np.float64) == q
    tol = np.where(exact, 0.0, G * U * np.abs(q))
    return np.floor(q - tol), np.floor(q + tol)


def contact64(pos, vel, colliders, dt, h, r, dt_step=None, mutant=None):
    """pos, vel: (N, 3) float32 at the start of the substep (all fluids, global original order); colliders: dicts (kind,
    params, rotation, translation, body, linvel, angvel, world_com) in slot order; dt: the lagging dt; dt_step: the step's
    dt (used by the current_dt mutant only)."""
    P0 = _f64(pos)
    V0 = _f64(vel)
    N = len(P0)
    p, v = P0.copy(), V0.copy()
    ep, ev = np.zeros((N, 3)), np.zeros((N, 3))
    excluded = np.zeros(N, bool)
    h = float(F(h))
    cut = 1.5 * h
    margin = 0.1 * float(F(r))
    dtp = float(F(dt_step if (mutant == "current_dt" and dt_step is not None) else dt))
    loosen = 0.0 if mutant == "aabb_not_loosened" else cut
    c_lo, c_hi = _cell_range(P0, h)
    res = Contact()
    res.samples = [None] * len(colliders)
    res.branches = {k: dict.fromkeys(BRANCHES, 0) for k in (BALL, CUBOID, CAPSULE)}
    res.reasons = {}
    res.candidates = 0
    res.processed = [None] * len(colliders)
    order = list(range(len(colliders)))
    if mutant == "reverse_slot_order":
        order = order[::-1]

    def exclude(mask, idx, reason):
        n = int((mask & ~excluded[idx]).sum())
        if n:
            res.reasons[reason] = res.reasons.get(reason, 0) + n
        excluded[idx[mask]] = True

    for k in order:
        col = colliders[k]
        kind = col["kind"]
        br = res.branches[kind]
        prm = np.zeros(3)
        prm[:len(col["params"])] = _f64(col["params"])
        R = _f64(col.get("rotation", np.eye(3))).reshape(3, 3)
        t = _f64(col.get("translation", (0, 0, 0)))
        perm = _signed_perm(R)
        ext = posed_ext(col, mutant)
        mins, maxs = t - ext - loosen, t + ext + loosen
        e_box = G * U * (3 * ext + 2 * (np.abs(t) + ext + cut) + cut)
        # box keys: each face key may be either of the floors within its bound
        lo_q, hi_q = mins / h, maxs / h
        lo_tol, hi_tol = e_box / h + G * U * np.abs(lo_q), e_box / h + G * U * np.abs(hi_q)
        klo = (np.floor(lo_q - lo_tol), np.floor(lo_q + lo_tol))
        khi = (np.floor(hi_q - hi_tol), np.floor(hi_q + hi_tol))
        sure_in = np.all((c_lo >= klo[1]) & (c_hi <= khi[0]), axis=1)
        sure_out = np.any((c_hi < klo[0]) | (c_lo > khi[1]), axis=1)
        in_box = np.all((np.floor(P0 / h) >= np.floor(lo_q)) & (np.floor(P0 / h) <= np.floor(hi_q)), axis=1)
        if mutant == "start_state":
            p_use, v_use, ep_use, ev_use = P0, V0, np.zeros_like(ep), np.zeros_like(ev)
        else:
            p_use, v_use, ep_use, ev_use = p, v, ep, ev
        pr_all = p_use if mutant == "current_position" else p_use + v_use * dtp
        # prediction bound: the exact rounding of fl(p + fl(v dt)) where p and v are exactly known
        known = np.all((ep_use == 0) & (ev_use == 0), axis=1)
        p32, v32 = p_use.astype(F), v_use.astype(F)
        f32 = (p32 if mutant == "current_position" else p32 + v32 * F(dtp)).astype(np.float64)
        e_gen = ep_use + ev_use * dtp + G * U * (2 * np.abs(v_use) * dtp + np.abs(p_use))
        e_pr_all = np.where(known[:, None], np.abs(f32 - pr_all), e_gen)
        s_box = np.minimum(pr_all - mins, maxs - pr_all)
        tol_box = e_pr_all + e_box
        aabb = np.all(s_box >= 0, axis=1)
        aabb_sure_out = np.any(s_box < -tol_box, axis=1)
        aabb_sure_in = np.all(s_box > tol_box, axis=1)
        maybe = ~sure_out & ~aabb_sure_out
        br["cell_outside"] += int((~in_box & aabb).sum())
        res.candidates += int(in_box.sum())
        exclude((~sure_in | ~aabb_sure_in) & maybe, np.arange(N), "cell_or_aabb")
        br["prediction_outside"] += int((in_box & ~aabb).sum())
        idx = np.nonzero(in_box & aabb)[0]
        # excluded particles may still be sampled wherever their (exact) start cell may lie in the box
        amb_extra = np.nonzero(~sure_out & excluded & ~(in_box & aabb))[0]
        pr, e_pr = pr_all[idx], e_pr_all[idx]
        pi, vi, epi, evi = p_use[idx], v_use[idx], ep_use[idx], ev_use[idx]
        # local frame l = R^T (pr - t)
        w = pr - t
        e_w = _rn(w, e_pr)
        Rt = R if mutant == "r_for_rt" else R.T
        l = w @ Rt.T
        e_l = e_w @ np.abs(Rt).T
        if not perm:
            e_l = e_l + G * 3 * U * (np.abs(w) @ np.abs(Rt).T)
        nel = np.linalg.norm(e_l, axis=1)
        m = len(idx)
        amb = np.zeros(m, bool)
        valid = np.ones(m, bool)
        q = np.zeros((m, 3))
        eq = np.zeros((m, 3))
        if kind == BALL:
            rb = prm[0]
            nl = np.linalg.norm(l, axis=1)
            centre = nl == 0
            valid = ~centre
            br["ball_centre"] += int(centre.sum())
            amb_centre = ~centre & (nl <= G * nel)
            nls = np.where(centre, 1.0, nl)
            inside = nl <= rb
            amb_in = _near(nl - rb, G * (nel + 2.5 * U * np.maximum(nl, rb)))
            q = l * (rb / nls)[:, None]
            eq = (2 * G * rb * nel / nls)[:, None] + 5 * G * U * rb + 0 * l
            amb_geo = amb_centre
        elif kind == CUBOID:
            e = prm
            mp, pm = -e - l, l - e
            tmp, tpm = _rn(mp, e_l), _rn(pm, e_l)
            six = np.concatenate([mp, pm], axis=1)
            tsix = np.concatenate([tmp, tpm], axis=1)
            top = six.max(axis=1)
            inside = top <= 0
            amb_in = _near(top, tsix[np.arange(m), six.argmax(axis=1)])
            # nearest face: per axis the larger of (mp, pm), a tie to the mins face; across axes the first maximum
            cand_max = (mp < pm) if mutant != "ties_to_maxs" else (mp <= pm)
            val = np.where(cand_max, pm, mp)
            a_id = val.argmax(axis=1)
            is_max = cand_max[np.arange(m), a_id]
            qin = l.copy()
            qin[np.arange(m), a_id] = np.where(is_max, e[a_id], -e[a_id])
            qout = np.clip(l, -e, e)
            q = np.where(inside[:, None], qin, qout)
            eq = e_l + 2 * G * U * (e + np.abs(l))
            srt = np.sort(six, axis=1)
            order6 = np.argsort(six, axis=1)
            t1 = tsix[np.arange(m), order6[:, -1]]
            t2 = tsix[np.arange(m), order6[:, -2]]
            amb_geo = (inside | amb_in) & _near(srt[:, -1] - srt[:, -2], t1 + t2) & (srt[:, -1] < -t1)
        else:
            a, rc = prm[0], prm[1]
            cy = np.clip(l[:, 1], -a, a)
            dvec = np.stack([l[:, 0], l[:, 1] - cy, l[:, 2]], axis=1)
            dn = np.linalg.norm(dvec, axis=1)
            axis_ = dn == 0
            br["capsule_axis"] += int(axis_.sum())
            dns = np.where(axis_, 1.0, dn)
            inside = dn <= rc
            amb_in = _near(dn - rc, G * (nel + 3 * U * np.maximum(dn, rc)))
            s = rc / dns
            q = np.stack([np.where(axis_, rc, l[:, 0] * s), np.where(axis_, cy, cy + dvec[:, 1] * s), np.where(axis_, 0.0, l[:, 2] * s)], axis=1)
            eq = (2 * G * rc * nel / dns)[:, None] + 5 * G * U * rc + 0 * l
            eq[:, 1] += e_l[:, 1] + G * U * (np.abs(cy) + rc)
            eq = np.where(axis_[:, None], np.stack([np.zeros(m), e_l[:, 1], np.zeros(m)], axis=1), eq)
            amb_geo = (~axis_ & (dn <= G * nel)) | _near(np.abs(l[:, 1]) - a, e_l[:, 1])
        # world projection qw = R q + t, d = pr - qw
        qw = q @ R.T + t
        e_qw = eq @ np.abs(R).T + G * U * np.abs(qw)
        if not perm:
            e_qw = e_qw + G * 3 * U * (np.abs(q) @ np.abs(R).T)
        d = pr - qw
        e_d = e_pr + e_qw + G * U * np.abs(d)
        ned = np.linalg.norm(e_d, axis=1)
        depth = np.linalg.norm(d, axis=1)
        e_depth = G * (ned + 2.5 * U * depth)
        has_n = depth > EPS32
        amb_eps = _near(depth - EPS32, e_depth)
        maybe_n = has_n | amb_eps
        deps = np.where(depth > 0, depth, 1.0)
        n = d / deps[:, None]
        e_n = (2 * G * ned / deps)[:, None] + 3 * G * U + 0 * d
        push = valid & has_n & inside
        ve = np.sum(n * vi, axis=1)
        e_ve = np.sum(np.abs(vi) * e_n + np.abs(n) * evi, axis=1) + 3 * G * U * np.sum(np.abs(n * vi), axis=1)
        gate = ve > 0 if mutant != "no_vn_gate" else np.ones(m, bool)
        amb_ve = push & _near(ve, e_ve) & (mutant != "no_vn_gate")
        cut_on = mutant != "no_cut"
        beyond = valid & has_n & ~inside & (depth > cut) & cut_on
        amb_cut = valid & maybe_n & ~inside & _near(depth - cut, e_depth + U * cut) & cut_on
        amb = valid & ((amb_eps & (inside | amb_in)) | (maybe_n & amb_in) | amb_ve | amb_cut) | amb_geo
        exclude(amb, idx, "projection")
        # pushes: p -= n (depth + margin); v -= n (n.v) when n.v > 0
        mg = 0.0 if mutant == "no_margin" else margin
        sdep = depth + mg
        e_s = e_depth + G * U * sdep + 2 * U * mg
        newp = pi - n * sdep[:, None]
        e_newp = epi + e_n * sdep[:, None] + np.abs(n) * e_s[:, None] + G * U * (np.abs(n) * sdep[:, None] + np.abs(newp))
        dv = push & gate
        newv = np.where(dv[:, None], vi - n * ve[:, None], vi)
        e_newv = np.where(dv[:, None], evi + e_n * np.abs(ve)[:, None] + np.abs(n) * e_ve[:, None]
                          + G * U * (np.abs(n * ve[:, None]) + np.abs(newv)), evi)
        p[idx[push]], ep[idx[push]] = newp[push], e_newp[push]
        v[idx[push]], ev[idx[push]] = newv[push], e_newv[push]
        emit = valid & ~beyond
        br["pushed"] += int(push.sum())
        br["shell"] += int((valid & has_n & ~inside & ~beyond).sum())
        br["beyond"] += int(beyond.sum())
        br["on_surface"] += int((valid & ~has_n).sum())
        if mutant == "local_point_velocity":
            sv, esv = body_velocity(q, eq, col)
        else:
            sv, esv = body_velocity(qw, e_qw, col)
        keep = emit | excluded[idx]
        sidx = np.concatenate([idx[keep], amb_extra])
        nx = len(amb_extra)
        nanx = np.full((nx, 3), np.nan)
        res.processed[k] = idx
        S = dict(idx=sidx, q=np.concatenate([qw[keep], nanx]), eq=np.concatenate([e_qw[keep], nanx]),
                 v=np.concatenate([sv[keep], nanx]), ev=np.concatenate([esv[keep], nanx]),
                 amb=np.concatenate([excluded[idx][keep], np.ones(nx, bool)]))
        o = np.argsort(S["idx"], kind="stable")
        res.samples[k] = {key: val[o] for key, val in S.items()}
    res.pos, res.vel, res.ep, res.ev, res.excluded = p, v, ep, ev, excluded
    res.n_samples = sum(int((~s["amb"]).sum()) for s in res.samples)
    res.n_pushes = int(np.any(p != P0, axis=1).sum())
    return res


def advance(res, dt):
    """update_positions with no velocity change (solver iterations 0, no gravity, no forces): P' = P + v dt, two roundings."""
    dt = float(F(dt))
    P = res.pos + res.vel * dt
    e = res.ep + res.ev * dt + G * U * (np.abs(res.vel) * dt + np.abs(P))
    return P, e


def ratio(got, ref, bound):
    err = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err == 0, 0.0, np.inf))


def check_fluid(res, P, V, dt):
    """Worst |err| / bound of the positions and velocities after the step, over the particles not excluded."""
    Pr, eP = advance(res, dt)
    keep = ~res.excluded
    rp = ratio(P, Pr, eP)[keep]
    rv = ratio(V, res.vel, res.ev)[keep]
    return float(rp.max(initial=0.0)), float(rv.max(initial=0.0))


def match_samples(S, sp, sv):
    """Walks the device samples (sp, sv in key order) and the reference S in original-index order: every sample of a
    particle not excluded must be present and within its bound; an excluded particle's may be present or absent.  Returns
    the worst |err| / bound (inf where the walk fails)."""
    sp, sv = np.asarray(sp, np.float64), np.asarray(sv, np.float64)
    amb = S["amb"]
    nref, m = len(amb), len(sp)
    worst = 0.0

    def fit(i, j):
        return max(float(ratio(sp[i], S["q"][j], S["eq"][j]).max()), float(ratio(sv[i], S["v"][j], S["ev"][j]).max()))

    i = j = 0
    while j < nref:
        if not amb[j]:
            if i >= m:
                return np.inf
            r = fit(i, j)
            if not r <= 1.0:
                return max(r, 1.0 + 1e-9) if np.isfinite(r) else np.inf
            worst = max(worst, r)
            i += 1
            j += 1
            continue
        k = j
        while k < nref and amb[k]:
            k += 1
        run = k - j
        chosen = None
        for t_ in range(run + 1):
            if k == nref:
                if i + t_ == m:
                    chosen = t_
                    break
            elif i + t_ < m and fit(i + t_, k) <= 1.0:
                chosen = t_
                break
        if chosen is None:
            return np.inf
        i += chosen
        j = k
    return worst if i == m else np.inf


def static64(local, col, mutant=None):
    """StaticSampling (:180-191): world points R l + t and the body's velocity at the LOCAL point (:183), with bounds."""
    L = _f64(local)
    R = _f64(col.get("rotation", np.eye(3))).reshape(3, 3)
    t = _f64(col.get("translation", (0, 0, 0)))
    x = L @ R.T + t
    ex = G * U * (3 * (np.abs(L) @ np.abs(R).T) + np.abs(x))
    at, eat = (x, ex) if mutant == "world_point_velocity" else (L, np.zeros_like(L))
    v, evv = body_velocity(at, eat, col)
    return x, ex, v, evv


def impulse64(entries, dt, dt_prev=None, nb_total=None, mutant=None):
    """transmit_forces (:263-287).  entries: one dict per collider (slot, bslot, body, world_com, translation, positions,
    forces; forces and positions in the same order, read back from the world).  Returns {slot: (lin, ang, e_lin, e_ang)}.
    nb_total: the world's boundary particle count (sizes k_collider_impulse's grid: min(ceil(B / 256), 264) blocks of 256,
    each summing its strided slots)."""
    dt = float(F(dt_prev if mutant == "lagging_dt" else dt))
    out = {}
    dropped = max((e["bslot"] for e in entries if e.get("body") == BODY_DYNAMIC), default=None) if mutant == "drop_boundary_slot" else None
    for e in entries:
        body = e.get("body", BODY_NONE)
        counted = body == BODY_DYNAMIC or (mutant == "fixed_counted" and body == BODY_FIXED)
        f = _f64(e["forces"]).reshape(-1, 3)
        if not counted or len(f) == 0 or e["bslot"] == dropped:
            out[e["slot"]] = (np.zeros(3), np.zeros(3), np.zeros(3), np.zeros(3))
            continue
        x = _f64(e["positions"]).reshape(-1, 3)
        com = _f64(e["translation"] if mutant == "torque_about_translation" else e["world_com"])
        fdt = f * dt
        rr = x - com
        lin = fdt.sum(axis=0)
        ang = np.cross(rr, fdt).sum(axis=0)
        B = max(int(nb_total if nb_total is not None else len(f)), 1)
        blocks = min(-(-B // 256), 264)
        terms = min(len(f), 256 * -(-B // (256 * blocks)))
        e_lin = (terms + blocks + 2) * U * np.abs(fdt).sum(axis=0)
        e_ang = (terms + blocks + 5) * U * _cross_abs(rr, fdt).sum(axis=0)
        out[e["slot"]] = (lin, ang, e_lin, e_ang)
    return out


# ---- scenes: shared by the CPU checks of the float32 restatement and the GPU checks of the device ------------------------
def rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return (rz @ ry @ rx).astype(F)


RZ90 = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], F)   # signed permutations: their poses are exact
RX90 = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], F)


def lattice(n, spacing, origin, seed=None, amplitude=0.0):
    g = np.stack(np.meshgrid(*[np.arange(k) for k in n], indexing="ij"), axis=-1).reshape(-1, 3)
    pts = (np.asarray(origin, np.float64) + (g + 0.5) * spacing)
    if seed is not None:
        pts = pts + np.random.default_rng(seed).uniform(-amplitude, amplitude, pts.shape) * spacing
    return pts.astype(F)


def _state(t, R=None, body=BODY_NONE, linvel=(0, 0, 0), angvel=(0, 0, 0), com=None):
    t = np.asarray(t, F)
    return dict(translation=t, rotation=np.eye(3, dtype=F) if R is None else np.asarray(R, F), body=body, linvel=np.asarray(linvel, F),
                angvel=np.asarray(angvel, F), world_com=t.copy() if com is None else np.asarray(com, F))


def _overlap_states(k):
    """Slot order: a dynamic ball (identity rotation, dyadic pose), a rotated dynamic cuboid and a rotated dynamic capsule
    whose loosened AABBs overlap pairwise, a fixed cuboid and a parentless capsule with signed-permutation rotations."""
    return [_state((0.3125, 0.3125 - k / 256.0, 0.3125), body=BODY_DYNAMIC, linvel=(0, -1, 0), angvel=(0.5, 2, -1)),
            _state((0.45, 0.28, 0.33), rot(0.3 + 0.1 * k, 0.2, 0.5), BODY_DYNAMIC, (0.3, 0, 0.1), (0, 1.5, 2), (0.4, 0.3, 0.33)),
            _state((0.2, 0.42, 0.56), rot(0.7, -0.4 + 0.05 * k, 0.9), BODY_DYNAMIC, (0, 0, 0), (-1, 0, 3), (0.2, 0.4, 0.56)),
            _state((0.75, 0.5, 0.25), RZ90, BODY_FIXED, (0.25, 0, 0), (0, 0, 1)),
            _state((0.25, 0.75, 0.75), RX90, BODY_NONE, (1, 1, 1), (1, 1, 1))]


OVERLAP_SHAPES = [(BALL, (0.125,)), (CUBOID, (0.2, 0.08, 0.14)), (CAPSULE, (0.12, 0.07)), (CUBOID, (0.125, 0.0625, 0.1875)),
                  (CAPSULE, (0.125, 0.0625))]


def _overlap():
    R = 0.05
    h = float(F(R) * F(2) * F(2))
    rng = np.random.default_rng(3)
    a = lattice((9, 8, 9), R * 1.9, (0.05, 0.08, 0.05), seed=3, amplitude=0.2)
    va = rng.normal(0, 3.0, a.shape).astype(F)
    b = (rng.random((300, 3)) * np.array([0.8, 0.7, 0.8]) + np.array([0.0, 0.05, 0.0])).astype(F)
    vb = rng.normal(0, 2.0, b.shape).astype(F)
    st = _overlap_states(0)
    # exact geometry, at rest: the ball's centre and a point on its surface; a point on a face of the fixed cuboid and its
    # centre (a tie between the two y faces, which goes to the mins face); a point on the parentless capsule's axis and one on
    # its surface
    exact = [st[0]["translation"], st[0]["translation"] + F(0.125) * np.array([0, 0, -1], F)]
    for (kind, prm), s, locs in ((OVERLAP_SHAPES[3], st[3], [(0.125, 0.03125, 0.0625), (0, 0, 0)]),
                                 (OVERLAP_SHAPES[4], st[4], [(0, 0.0625, 0), (0.0625, -0.03125, 0)])):
        for l in locs:
            exact.append(s["rotation"] @ np.asarray(l, F) + s["translation"])
    ex = np.asarray(exact, F)
    # per collider, one fast particle whose cell lies one cell below its box while, after a step of DT, its prediction over
    # the next step of DT lies inside its AABB (not a candidate: cell_outside)
    fast, vfast = [], []
    DT = 0.004
    for (kind, prm), s in zip(OVERLAP_SHAPES, st):
        col = dict(kind=kind, params=prm, **s)
        mins = s["translation"].astype(np.float64) - posed_ext(col) - 1.5 * h
        p1 = np.floor(mins[0] / h) * h - 0.25 * h
        vx = (mins[0] + 0.3 * h - p1) / DT
        fast.append((p1 - vx * DT, s["translation"][1] + 0.013, s["translation"][2] - 0.011))
        vfast.append((vx, 0.0, 0.0))
    b = np.concatenate([b, ex, np.asarray(fast, F)])
    vb = np.concatenate([vb, np.zeros_like(ex), np.asarray(vfast, F)])
    return dict(radius=R, fluids=[dict(positions=a, velocities=va, memberships=1, filter=1), dict(positions=b, velocities=vb)],
                shapes=OVERLAP_SHAPES, boundary_of_slot=[3, 5, 1, 2, 4], plain=True, states=_overlap_states, steps=6)


def _overflow():
    """A 0.4 m cuboid and a ball inside a block of 31^3 particles of radius 0.01: more than 4096 samples and pushes."""
    R = 0.01
    a = lattice((31, 31, 31), R * 1.9, (0.0, 0.0, 0.0), seed=5, amplitude=0.2)
    va = np.random.default_rng(5).normal(0, 0.3, a.shape).astype(F)

    def states(k):
        return [_state((0.3, 0.29 + 0.002 * k, 0.3), rot(0.2, 0.1 * k, 0.3), BODY_DYNAMIC, (0, 0.5, 0), (0, 1, 0), (0.31, 0.29, 0.3)),
                _state((0.42, 0.45, 0.44), None, BODY_DYNAMIC, (0, 0, -0.5), (1, 0, 0))]
    return dict(radius=R, fluids=[dict(positions=a, velocities=va)], shapes=[(CUBOID, (0.2, 0.2, 0.2)), (BALL, (0.12,))],
                boundary_of_slot=[0, 1], plain=False, states=states, steps=3)


def _dense_bin_and_clipping():
    """A clump of 96 particles in one cell inside a ball; a capsule whose cell box is clipped by the grid; a cuboid whose
    box lies outside it; a long diagonal capsule whose box covers all of it."""
    R = 0.05
    rng = np.random.default_rng(7)
    a = lattice((8, 6, 8), R * 1.9, (0.0, 0.0, 0.0), seed=7, amplitude=0.2)
    va = rng.normal(0, 1.0, a.shape).astype(F)
    clump = (np.array([0.41, 0.21, 0.41]) + rng.random((96, 3)) * 0.17).astype(F)  # one cell of h = 0.2: [0.4, 0.6)^2 x [0.2, 0.4)
    vc = rng.normal(0, 1.0, clump.shape).astype(F)

    def states(k):
        return [_state((0.5, 0.3, 0.5), None, BODY_DYNAMIC, (0, 0, 0), (0, 0, 3)),
                _state((0.02, 0.55, 0.7), rot(0.4, 0.3, 0.2 + 0.1 * k), BODY_DYNAMIC, (0.1, 0, 0), (0, 1, 0)),
                _state((4.0, 4.0, 4.0), rot(0.1, 0.2, 0.3), BODY_DYNAMIC),
                _state((0.4, 0.3, 0.4), rot(0.6, 0.5, 0.7), BODY_NONE)]
    return dict(radius=R, fluids=[dict(positions=np.concatenate([a, clump]), velocities=np.concatenate([va, vc]))],
                shapes=[(BALL, (0.15,)), (CAPSULE, (0.2, 0.08)), (CUBOID, (0.1, 0.1, 0.1)), (CAPSULE, (3.0, 0.05))],
                boundary_of_slot=[0, 1, 2, 3], plain=False, states=states, steps=4)


def _high_slot():
    """Contact colliders at collider slots 0 and 63 (the key's 6-bit slot field), on boundaries 5 and 63 of 64."""
    R = 0.05
    a = lattice((8, 6, 8), R * 1.9, (0.0, 0.0, 0.0), seed=11, amplitude=0.2)
    va = np.random.default_rng(11).normal(0, 1.0, a.shape).astype(F)

    def states(k):
        return [_state((0.3, 0.3, 0.3), rot(0.2, 0.3, 0.1 * k), BODY_DYNAMIC, (0, 1, 0), (1, 0, 0)),
                _state((0.5, 0.28, 0.5), rot(0.5, 0.1, 0.2), BODY_DYNAMIC, (0, 0, 1), (0, 2, 0))]
    return dict(radius=R, fluids=[dict(positions=a, velocities=va)], shapes=[(CUBOID, (0.15, 0.1, 0.12)), (CAPSULE, (0.1, 0.08))],
                slots=[0, 63], boundary_of_slot=[5, 63], plain=False, states=states, steps=3)


SCENES = dict(overlap=_overlap, overflow=_overflow, dense_bin_and_clipping=_dense_bin_and_clipping, high_slot=_high_slot)
DTS = (0.004, 0.008, 0.004 / 3)


def colliders_at(sc, k):
    return [dict(kind=kind, params=prm, **s) for (kind, prm), s in zip(sc["shapes"], sc["states"](k))]


def check_restatement(res, p32, v32, samples):
    """Worst |err| / bound of a float32 contact pass (pushed state and samples, in the reference's collider order) against
    the reference: dict(pushed_positions, pushed_velocities, samples)."""
    keep = ~res.excluded
    w = dict(pushed_positions=float(ratio(p32, res.pos, res.ep)[keep].max(initial=0.0)),
             pushed_velocities=float(ratio(v32, res.vel, res.ev)[keep].max(initial=0.0)))
    w["samples"] = max([match_samples(S, sp, sv) for S, (sp, sv) in zip(res.samples, samples)], default=0.0)
    return w


def run_reference(sc, step=None):
    """The scene's steps on the float64 reference alone (P' = P + v dt after each contact pass), as the GPU test steps the
    device.  step(k, pos, vel, res) is called with each step's input and reference.  Returns the per-step results."""
    pos = np.concatenate([f["positions"] for f in sc["fluids"]])
    vel = np.concatenate([f["velocities"] for f in sc["fluids"]])
    h = float(F(sc["radius"]) * F(2) * F(2))
    lag, out = 0.0, []
    for k in range(sc["steps"]):
        dt = DTS[k % len(DTS)]
        res = contact64(pos, vel, colliders_at(sc, k), lag, h, sc["radius"])
        if step is not None:
            step(k, pos, vel, res)
        out.append(res)
        P, _ = advance(res, dt)
        pos, vel = P.astype(F), res.vel.astype(F)
        lag = dt
    return out
