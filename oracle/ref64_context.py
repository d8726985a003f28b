"""What a host NonPressureForce receives (sph_host_force_ctx, include/sph.h), checked against oracle/ref64.py.

TEST INFRASTRUCTURE ONLY.  LiquidWorld.push_host_force2 hands solve(ctx) views that live for the call; `capture` copies
them.  `check` compares one captured ctx with the world's state around the step that made it:

  csr          offsets[0] == 0, never decreasing, per-particle lengths equal to num_fluid_contacts / num_boundary_contacts;
  membership   per particle, the multiset of (j_model, j) equals the reference's float32-test contacts over every fluid
               (boundary) under the interaction groups, each mapped to (object slot, index inside the object); the self
               contact (fluid_index, i) appears exactly once.  The order inside a particle is not pinned;
  weight       W_kd(r) and gradient g_kg(r) x_ij per component, within their bounds, x_ij rebuilt through the ctx's own
  gradient     indices: ctx.positions[i] - (the fluid's positions before the step)[j_model][j], or
               - ctx.boundaries[j_model].positions[j].  The gradient is exactly 0 where d^2 is at or below its zero
               threshold; contacts within 8u of that threshold are excluded and counted;
  views        positions, velocities, densities and volumes bit for bit against what the caller expects;
  acc_in       the accelerations on entry bit for bit against a twin world's (one whose plugin adds the same through the
               callback without contacts or boundaries, so that both stay on one trajectory);
  boundaries   per slot n, positions, velocities and volumes bit for bit against read_boundary_particles /
               read_boundary after the step, and the volumes within boundary_volume_sum's bound;
  scalars      kernel_radius, particle_radius, fluid, fluid_index and density0; NULL contacts / boundaries when not asked.

`check_acc_out` compares the accelerations after the step with the entry plus what the plugin added (a float32 add, bit for
bit) on the plugin's fluid and with the twin's everywhere else.

Error bounds, per contact (one term: n = 1 in Ref.bound's (n + c) u A + K).  ref64.kernel's kerr already carries the
argument's error (8u in r) and the polynomial's roundings (8u of its absolute value); beyond those:
  weight       sigma * poly: 1; margin 1                                                       C_WEIGHT   = C_NORM + 2
  gradient     inv_r from rsqrt.approx (2.2) of d2 (its 2u halve: 1), dsigma6 * inv_r 1, * poly 1, poly's q = r inv_h
               taken apart from inv_r 1, g * dx 1, dx = x_i - x_j 1; margin 1.8              C_GRADIENT = C_NORM + 10
The generic library's IEEE sqrt and divisions (kernel_dw_kind(r) / r: 1 more) stay below the same counts.
"""
from dataclasses import dataclass, field

import numpy as np

from . import ref64
from .ref64 import C_NORM, F, U
from .ref64_stages import passes_for

C_WEIGHT = C_NORM + 2
C_GRADIENT = C_NORM + 10
MAX_SLOTS = 64   # MAX_FLUIDS, MAX_BOUNDARIES <= 64


def capture(ctx):
    """A copy of everything solve(ctx) was handed (its arrays are freed when solve returns)."""
    cp = lambda a: None if a is None else np.array(a, copy=True)  # noqa: E731

    def contacts(c):
        if c is None:
            return None
        return dict(offsets=cp(c.offsets).astype(np.int64), j=cp(c.j), j_model=cp(c.j_model), weight=cp(c.weight), gradient=cp(c.gradient))

    return dict(dt=ctx.dt, inv_dt=ctx.inv_dt, kernel_radius=ctx.kernel_radius, particle_radius=ctx.particle_radius, fluid=ctx.fluid,
                fluid_index=ctx.fluid_index, density0=ctx.density0, n=len(ctx.positions), positions=cp(ctx.positions),
                velocities=cp(ctx.velocities), densities=cp(ctx.densities), volumes=cp(ctx.volumes), accelerations=cp(ctx.accelerations),
                ff=contacts(ctx.fluid_fluid_contacts), fb=contacts(ctx.fluid_boundaries_contacts),
                boundaries=None if ctx.boundaries is None else [{k: cp(v) for k, v in b.items()} for b in ctx.boundaries])


@dataclass
class State:
    """The world around one step, per object SLOT (a removed slot: alive False, no particles).
    fluids: dicts of positions (before the step), volumes (what the fluid holds), density0, memberships, filter.
    boundaries: dicts of positions, velocities, volumes (after the step: this step's particles), memberships, filter."""
    radius: float
    fluids: list
    boundaries: list
    kw: int = 0
    kg: int = 0
    _ps: object = field(default=None, repr=False)

    def passes(self):
        if self._ps is None:
            sc = dict(particle_radius=self.radius,
                      fluids=[dict(positions=np.asarray(f["positions"], F).reshape(-1, 3), volumes=f["volumes"], density0=f["density0"],
                                   memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF)) for f in self.fluids],
                      boundaries=[dict(positions=np.asarray(b["positions"], F).reshape(-1, 3), memberships=b.get("memberships", 1),
                                       filter=b.get("filter", 0xFFFFFFFF)) for b in self.boundaries])
            self._ps = passes_for(sc, kw=self.kw, kg=self.kg)
        return self._ps

    def offsets(self, objs):
        return np.r_[0, np.cumsum([len(o["positions"]) for o in objs])].astype(np.int64)


class Report:
    """Worst |err| / bound per value check, mismatching particles (or slots) per exact check, exclusions per check."""

    def __init__(self):
        self.worst, self.bad, self.excluded = {}, {}, {}

    def ratio(self, name, r):
        self.worst[name] = max(self.worst.get(name, 0.0), float(np.max(r)) if np.size(r) else 0.0)

    def exact(self, name, bad):
        bad = [int(x) for x in np.atleast_1d(bad)]
        self.bad.setdefault(name, [])
        self.bad[name] += bad

    def flagged(self):
        out = {k: v for k, v in self.worst.items() if not v <= 1.0}
        out.update({k: v[:8] for k, v in self.bad.items() if v})
        return out


def _bitwise_rows(a, b):
    """Rows where two float32 arrays differ in any bit (shape mismatch: every row, or [-1] when one side is empty)."""
    a, b = np.asarray(a, F), np.asarray(b, F)
    if a.shape != b.shape:
        return np.arange(max(len(a), len(b), 1)) if len(a) and len(b) else np.array([-1])
    d = a.view(np.uint32) != b.view(np.uint32)
    return np.nonzero(d.reshape(len(d), -1).any(axis=1))[0] if d.size else np.zeros(0, np.int64)


def reference_contacts(st, fluid, which):
    """The reference's contacts of fluid `fluid`'s particles as (i local, j_model, j local, x_ij float64)."""
    ps = st.passes()
    pr = ps.ff if which == "ff" else ps.fb
    fo = st.offsets(st.fluids)
    oo = fo if which == "ff" else st.offsets(st.boundaries)
    sel = (pr.i >= fo[fluid]) & (pr.i < fo[fluid + 1])
    jm = np.searchsorted(oo, pr.j[sel], side="right") - 1
    return pr.i[sel] - fo[fluid], jm, pr.j[sel] - oo[jm], pr.x[sel]


def _keys(i, jm, j, M):
    jm = np.minimum(np.asarray(jm, np.int64), MAX_SLOTS)
    j = np.minimum(np.asarray(j, np.int64), M - 1)
    return (np.asarray(i, np.int64) * (MAX_SLOTS + 1) + jm) * M + j


def _check_list(rep, cap, st, fluid, which, counts, exp_P, exp_B):
    c = cap[which]
    n = cap["n"]
    off = c["offsets"]
    objs = st.fluids if which == "ff" else st.boundaries
    sizes = np.array([len(o["positions"]) for o in objs], np.int64)
    # CSR shape
    if len(off) != n + 1 or off[0] != 0 or (np.diff(off) < 0).any() or off[-1] != len(c["j"]):
        rep.exact(which + "_csr", [-1])
        return
    rep.exact(which + "_csr", [] if counts is None else np.nonzero(np.diff(off) != np.asarray(counts, np.int64))[0])
    i_of = np.repeat(np.arange(n), np.diff(off))
    jm, j = c["j_model"].astype(np.int64), c["j"].astype(np.int64)
    # membership: per particle, the multiset of (j_model, j)
    ri, rjm, rj, _ = reference_contacts(st, fluid, which)
    M = int(max(sizes.max(initial=0), 1)) + 1
    k1 = np.sort(_keys(i_of, jm, j, M))
    k2 = np.sort(_keys(ri, rjm, rj, M))
    if not np.array_equal(k1, k2):
        u = np.union1d(k1, k2)
        c1 = np.searchsorted(k1, u, "right") - np.searchsorted(k1, u, "left")
        c2 = np.searchsorted(k2, u, "right") - np.searchsorted(k2, u, "left")
        rep.exact(which + "_membership", np.unique(u[c1 != c2] // (M * (MAX_SLOTS + 1))))
    else:
        rep.exact(which + "_membership", [])
    if which == "ff":
        self_ = np.bincount(i_of[(jm == cap["fluid_index"]) & (j == i_of)], minlength=n)
        rep.exact("ff_self", np.nonzero(self_ != 1)[0])
    # values at the valid entries, x_ij through the ctx's own indices
    valid = (jm < len(objs)) & (j < sizes[np.minimum(jm, len(objs) - 1)]) if len(objs) else np.zeros(len(j), bool)
    rep.excluded[which + "_invalid_index"] = rep.excluded.get(which + "_invalid_index", 0) + int((~valid).sum())
    src = exp_P if which == "ff" else exp_B
    xj = np.zeros((len(j), 3))
    for m in np.unique(jm[valid]):
        s = valid & (jm == m)
        xj[s] = np.asarray(src[m], F)[j[s]].astype(np.float64)
    xi = np.asarray(cap["positions"], F).astype(np.float64)[i_of]
    x = (xi - xj)[valid]
    d2 = (x * x).sum(1)
    r = np.sqrt(d2)
    h = float(F(st.passes().h))
    w, wa, we = ref64.kernel(st.kw, "w", r, h)
    wb = (1 + C_WEIGHT) * U * wa + we
    rep.ratio(which + "_weight", _ratio(c["weight"][valid], w, wb))
    g, ga, ge = ref64.kernel(st.kg, "g", r, h)
    t = ref64.grad_threshold(st.kg, h)
    zero = d2 <= t
    g, ga, ge = np.where(zero, 0.0, g), np.where(zero, 0.0, ga), np.where(zero, 0.0, ge)
    ax = np.abs(x)
    gref = g[:, None] * x
    gb = ((1 + C_GRADIENT) * U * ga + ge)[:, None] * ax
    amb = np.abs(d2 - t) <= 8 * U * t
    rr = _ratio(c["gradient"][valid], gref, gb).max(axis=1, initial=0.0) if len(x) else np.zeros(0)
    rep.ratio(which + "_gradient", np.where(amb, 0.0, rr))
    rep.excluded[which + "_gradient"] = rep.excluded.get(which + "_gradient", 0) + int(amb.sum())


def _ratio(gpu, ref, bound):
    err = np.abs(np.asarray(gpu, np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err == 0, 0.0, np.inf))


def check(cap, st, fluid, expect, rep=None):
    """Compare one captured ctx of fluid slot `fluid` with the state around its step.  expect: dict with
      velocities, densities, volumes, acc_in (float32 arrays the ctx must equal bit for bit; any may be missing),
      counts_ff, counts_fb (the per-particle list lengths), handle, density0, particle_radius, h,
      contacts, boundaries (the flags the force was pushed with),
      boundary_n (per slot: read_boundary's count, 0 for a removed slot).
    Returns the Report (a new one unless rep is given)."""
    rep = Report() if rep is None else rep
    ps = st.passes()
    # scalars and flags
    sc = []
    if cap["kernel_radius"] != F(expect["h"]):
        sc.append(0)
    if cap["particle_radius"] != F(expect["particle_radius"]):
        sc.append(1)
    if cap["fluid"] != expect["handle"] or cap["fluid_index"] != fluid:
        sc.append(2)
    if cap["density0"] != F(expect["density0"]):
        sc.append(3)
    if (cap["ff"] is None) == bool(expect["contacts"]) or (cap["fb"] is None) == bool(expect["contacts"]):
        sc.append(4)
    if (cap["boundaries"] is None) == bool(expect["boundaries"]):
        sc.append(5)
    rep.exact("scalars", sc)
    # particle views, bit for bit
    rep.exact("positions", _bitwise_rows(cap["positions"], st.fluids[fluid]["positions"]))
    for name in ("velocities", "densities", "volumes"):
        if expect.get(name) is not None:
            rep.exact(name, _bitwise_rows(cap[name], expect[name]))
    if expect.get("acc_in") is not None:
        rep.exact("acc_in", _bitwise_rows(cap["accelerations"], expect["acc_in"]))
    # boundary views
    exp_B = [np.asarray(b["positions"], F).reshape(-1, 3) for b in st.boundaries]
    if cap["boundaries"] is not None:
        bad = [] if len(cap["boundaries"]) == len(st.boundaries) else [-1]
        for b, (v, e) in enumerate(zip(cap["boundaries"], st.boundaries)):
            if len(v["positions"]) != expect["boundary_n"][b]:
                bad.append(b)
                continue
            for k in ("positions", "velocities", "volumes"):
                if len(_bitwise_rows(v[k], e[k])):
                    bad.append(b)
                    break
        rep.exact("boundary_views", bad)
        if len(ps.BP) and not bad:
            vol = np.concatenate([np.asarray(v["volumes"], F) for v in cap["boundaries"]]).astype(np.float64)
            rep.ratio("boundary_volume", ref64.ratio(1.0 / vol, ps.boundary_volume_sum(), ref64.C_PASS["boundary_volume"]))
        ctx_B = [np.asarray(v["positions"], F).reshape(-1, 3) for v in cap["boundaries"]]
        if [len(p) for p in ctx_B] == [len(p) for p in exp_B]:
            exp_B = ctx_B
    # contacts
    if cap["ff"] is not None:
        exp_P = [np.asarray(f["positions"], F).reshape(-1, 3) for f in st.fluids]
        _check_list(rep, cap, st, fluid, "ff", expect.get("counts_ff"), exp_P, exp_B)
        _check_list(rep, cap, st, fluid, "fb", expect.get("counts_fb"), exp_P, exp_B)
    return rep


def check_acc_out(after, twin, entry, added, fluid, rep=None, name="acc_out"):
    """after / twin: per fluid slot, debug("acceleration") of the world and of its twin after the step; entry: the
    accelerations the plugin of slot `fluid` was handed, added: what it added.  Slot `fluid` must hold f32(entry + added)
    and every other slot the twin's, bit for bit (mismatching slots are reported)."""
    rep = Report() if rep is None else rep
    bad = []
    for k, (a, t) in enumerate(zip(after, twin)):
        want = (np.asarray(entry, F) + np.asarray(added, F)).astype(F) if k == fluid else t
        if len(_bitwise_rows(a, want)):
            bad.append(k)
    rep.exact(name, bad)
    return rep


def pattern(n, fluid, salt=0):
    """What a test plugin adds to its fluid's accelerations: distinct per particle index, fluid slot and plugin."""
    i = np.arange(n, dtype=np.float64)[:, None]
    k = np.array([1.0, -2.0, 3.0])[None, :]
    return (1e-3 * k * ((i % 17) + 1) * (fluid + 1 + 0.5 * salt)).astype(F)


def standin(st, fluid, velocities, densities, accelerations, boundaries=None):
    """A float32 ctx built from the reference: contacts in the reference's (i, j) order with f32 weights and gradients, the
    given particle views and the state's boundaries (boundaries: override the views, e.g. a stale pose)."""
    out = dict(dt=F(0.004), inv_dt=F(250.0), kernel_radius=F(st.passes().h), particle_radius=F(st.radius), fluid=fluid,
               fluid_index=fluid, density0=F(st.fluids[fluid]["density0"]), n=len(st.fluids[fluid]["positions"]),
               positions=np.asarray(st.fluids[fluid]["positions"], F).reshape(-1, 3).copy(), velocities=np.asarray(velocities, F).copy(),
               densities=np.asarray(densities, F).copy(), volumes=np.asarray(st.fluids[fluid]["volumes"], F).copy(),
               accelerations=np.asarray(accelerations, F).copy())
    h = float(F(st.passes().h))
    for which in ("ff", "fb"):
        i, jm, j, x = reference_contacts(st, fluid, which)
        r = np.sqrt((x * x).sum(1))
        w = ref64.kernel(st.kw, "w", r, h)[0]
        g = ref64.kernel(st.kg, "g", r, h)[0]
        g = np.where((x * x).sum(1) <= ref64.grad_threshold(st.kg, h), 0.0, g)
        off = np.r_[0, np.cumsum(np.bincount(i, minlength=out["n"]))].astype(np.int64)
        out[which] = dict(offsets=off, j=j.astype(np.uint32), j_model=jm.astype(np.uint32), weight=w.astype(F),
                          gradient=(g[:, None] * x).astype(F))
    bs = st.boundaries if boundaries is None else boundaries
    out["boundaries"] = [dict(positions=np.asarray(b["positions"], F).reshape(-1, 3).copy(),
                              velocities=np.asarray(b["velocities"], F).reshape(-1, 3).copy(),
                              volumes=np.asarray(b["volumes"], F).copy()) for b in bs]
    return out
