"""Feed each DFSPH gather pass its own inputs and check its output against oracle/ref64.py, particle by particle.

TEST INFRASTRUCTURE ONLY.  A world (salva_b200.LiquidWorld or oracle.OracleWorld: the same driving code checks both) is
replayed from scratch once per stage, with the loop shapes pinned by force_iterations(n_div, n_press) and gravity 0:
  (0, 0)  counts, boundary volumes, rho, alpha and the neighbour search's divergence sweep (v* = V0); the predicted density
          of the pressure loop's only evaluation; with Akinci2013, the unfused force passes;
  (1, 0)  one divergence update: read_fluid velocities = V0 - (the update's sum), kappa_i = f32(div_i alpha_i) from the
          float32 outputs of (0, 0), formed as the kernels form it; the evaluation after it (v* = those velocities); with
          Akinci2013 on a single uniform-mass fluid, the fused force (normals in the update, force in that evaluation);
  (1, 1)  one pressure update: velocity_change = f32(acc dt) - (the update's sum), kappa_i = max(f32(f32(rho*_i - rho0)
          alpha_i), 0) from the predicted densities of (1, 0);
  XSPH    forces see the previous step's inv_dt, 0 on the first step: step 1, then step 2 with (1, 0) (fused into the last
          evaluation for a single uniform-mass fluid) or (0, 0) (the separate pass), on positions P1, the velocities V2 the
          loop left and the densities of step 2.
Gating decisions (the 20-contact gate, the clamp, kappa > 0) are integer or sign decisions on the same float32 inputs, so the
reference takes them exactly as the kernels do.  Particles whose outcome hangs on a float decision inside the bound (alpha's
den <= 1e-5, a squared distance at the gradient's zero threshold) are excluded and counted.
"""
import numpy as np

from . import ref64
from .ref64 import C_PASS, F

R = 0.05
DT = 0.004
ZERO_G = (0.0, 0.0, 0.0)


# ---- scenes ------------------------------------------------------------------------------------------------------------------
def _lattice(nx, ny, nz, compress, seed, amplitude, origin=(0.0, 0.0, 0.0)):
    from salva_b200 import scenes
    return scenes.jitter(scenes.block_lattice(nx, ny, nz, R * compress, origin=origin), R, seed, amplitude=amplitude)


def _tank(nx, nz, compress, shift=(0.0, 0.0, 0.0), top=1.0):
    from salva_b200 import scenes
    s = np.asarray(shift, np.float64)
    t = scenes.open_tank(tuple(np.array([-R, -R, -R]) + s), tuple(np.array([nx * 2 * R * compress + R, top, nz * 2 * R * compress + R]) + s), R)
    return t.astype(F)


def _bvel(n, seed):
    rng = np.random.default_rng(seed)
    return (np.array([0.05, -0.1, 0.02], F) + rng.normal(0, 0.02, (n, 3))).astype(F)


def _fluid(pts, seed, density0=1000.0, **kw):
    rng = np.random.default_rng(seed)
    return dict(positions=pts.astype(F), velocities=rng.normal(0, 0.2, pts.shape).astype(F), density0=density0, **kw)


def scene_block(shift=(0.0, 0.0, 0.0)):
    """13 x 9 x 11 jittered block at 0.75 spacing (~2.4x rest density): lists longer than the staging rows (32 fluid, 8
    boundary) and the initial capacity of 64, every count mod 4; plus a sparse row along the floor, whose particles are
    below rest density (kappa = 0 under pressure) and touch the tank."""
    nx, ny, nz, c = 13, 9, 11, 0.75
    pts = _lattice(nx, ny, nz, c, 23, 0.4)
    row = np.stack([np.linspace(0.05, nx * 2 * R * c - 0.05, 12), np.full(12, 0.01), np.full(12, nz * 2 * R * c + 0.12)], 1)
    pts = np.concatenate([pts, row.astype(F)]) + np.asarray(shift, F)
    tank = _tank(nx, nz, c + 0.2 / nz, shift)
    return dict(fluids=[_fluid(pts.astype(F), 7)], boundaries=[dict(positions=tank, velocities=_bvel(len(tank), 3))])


def scene_far():
    """The block far from the origin: negative cell coordinates, and float32 coordinates as coarse as 2^-14 m."""
    return scene_block(shift=(1000.0, -1000.0, 513.0))


def scene_gate():
    """A sparse, strongly jittered block: about 20 contacts per particle, so n_f + n_b runs through 19, 20 and 21."""
    nx, ny, nz, c = 11, 10, 11, 1.2
    pts = _lattice(nx, ny, nz, c, 31, 0.6)
    tank = _tank(nx, nz, c)
    return dict(fluids=[_fluid(pts, 11)], boundaries=[dict(positions=tank, velocities=_bvel(len(tank), 5))])


def _exact_h_offset(h):
    """An x at which f32(x + h) - x == h exactly, so the pair (x, x + h) sits at d^2 = h^2 in float32."""
    for k in range(1, 4096):   # x in [1/8, 1/4): its ulp is h's, so x + h can be exact
        x = F(0.13 + k * 2.0 ** -26)
        y = F(x + F(h))
        if F(y - x) == F(h):
            return x, y
    raise AssertionError("no exact offset found")


def fma_flips(h, n, seed):
    """Pairs of float32 points whose unfused squared distance passes d^2 <= h^2 while the fused one (as the CUDA pair
    evaluation forms it) does not, found by search with an exact FMA emulation."""
    rng = np.random.default_rng(seed)
    h2 = F(F(h) * F(h))
    out = []
    while len(out) < n:
        a = (rng.uniform(0.3, 0.6, (4096, 3))).astype(F)
        u = rng.normal(size=(4096, 3))
        u /= np.linalg.norm(u, axis=1)[:, None]
        b = (a + u * float(h) * (1 + rng.uniform(-3e-7, 3e-7, (4096, 1)))).astype(F)
        d = ref64.f32_d2(a, b)
        cand = np.nonzero(np.abs(d.astype(np.float64) - float(h2)) <= 2 ** -22 * float(h2))[0]
        if len(cand) == 0:
            continue
        fd = ref64.fma_d2(a[cand], b[cand])
        hit = cand[(d[cand] <= h2) & (fd > h2)]
        out += [(a[k], b[k]) for k in hit]
    return out[:n]


def scene_pairs():
    """Pair edges inside a 2.3x compressed block: exactly coincident particles (d^2 = 0); pairs at 0 < d^2 <= eps^2 and
    at eps^2 < d^2 <= (1e-5 h)^2 (no gradient; Akinci's cohesion still acts above eps^2); pairs at exactly d^2 = h^2; pairs the
    unfused test accepts while the fused d^2 lies above h^2; and fluid particles nearly on a boundary particle."""
    nx, ny, nz, c = 8, 7, 8, 0.76
    pts = _lattice(nx, ny, nz, c, 41, 0.2)
    h = F(F(R) * F(2.0) * F(2.0))
    extra = [pts[5], pts[77] + F(0)]                                   # coincident with particles 5 and 77
    extra += [(pts[100] + np.array([5e-8, 0, 0], F)).astype(F)]        # d^2 ~ 2.5e-15 < eps^2
    extra += [(pts[150] + np.array([0, 6e-7, 0], F)).astype(F)]        # eps^2 < d^2 ~ 3.6e-13 < (1e-5 h)^2
    extra += [(pts[200] + np.array([0, 0, -4e-7], F)).astype(F)]
    x0, x1 = _exact_h_offset(h)
    base = pts[250].copy()
    p = base.copy()
    p[0] = x0
    q = p.copy()
    q[0] = x1
    extra += [p, q]
    for a, b in fma_flips(h, 3, 5):
        extra += [a, b]
    pts = np.concatenate([pts, np.asarray(extra, F)]).astype(F)
    tank = _tank(nx, nz, c)
    near = [(tank[k] + np.array([0, 4e-7, 0], F)).astype(F) for k in (40, 60)]   # just above two floor particles
    pts = np.concatenate([pts, np.asarray(near, F)]).astype(F)
    return dict(fluids=[_fluid(pts, 13)], boundaries=[dict(positions=tank, velocities=_bvel(len(tank), 7))])


def _pass_t():
    """Threads per block of the gather passes: SPH_PASS_T's default in sph_kernels.cuh, so the tail scenes follow it."""
    import os
    import re
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "salva_b200", "csrc", "sph_kernels.cuh")
    return int(re.search(r"#define SPH_PASS_T (\d+)", open(src).read()).group(1))


PASS_T = _pass_t()
TAILS = (1, 31, 32, 33, PASS_T - 1, PASS_T + 1)


def scene_tail(n):
    """n particles of a compressed block: partial warps and blocks of the gather passes (n = 1 is a lone particle, self-only)."""
    pts = _lattice(6, 6, 6, 0.8, 43, 0.2)[:n]
    if n == 1:
        pts = np.array([[0.3, 0.5, 0.3]], F)
    return dict(fluids=[_fluid(pts, 17)], boundaries=[dict(positions=_tank(6, 6, 0.8), velocities=_bvel(len(_tank(6, 6, 0.8)), 9))])


def scene_volumes():
    """Per-particle volumes (no uniform-mass records): the generic k_vel_divergence / k_vel_update path."""
    sc = scene_block()
    n = len(sc["fluids"][0]["positions"])
    rng = np.random.default_rng(19)
    sc["fluids"][0]["volumes"] = ((2 * R) ** 3 * rng.uniform(0.8, 1.2, n)).astype(F)
    return sc


def scene_two_fluids():
    """Two fluids with different rest densities and interaction groups: the floor meets both, the walls only fluid 0 and
    want their forces (the boundary-force kernel variants, whose per-particle forces are checked too)."""
    sc = scene_block()
    pts, vel = sc["fluids"][0]["positions"], sc["fluids"][0]["velocities"]
    up = pts[:, 0] > np.median(pts[:, 0])  # side by side: both fluids touch the floor
    tank = sc["boundaries"][0]
    floor = tank["positions"][:, 1] < -R / 2
    return dict(fluids=[dict(positions=pts[~up], velocities=vel[~up], density0=1000.0, memberships=1, filter=0xFFFFFFFF),
                        dict(positions=pts[up], velocities=vel[up], density0=800.0, memberships=2, filter=0xFFFFFFFF)],
                boundaries=[dict(positions=tank["positions"][floor], velocities=tank["velocities"][floor]),
                            dict(positions=tank["positions"][~floor], velocities=tank["velocities"][~floor], memberships=4,
                                 filter=1, want_forces=True)])


SCENES = dict(block=scene_block, far=scene_far, gate=scene_gate, pairs=scene_pairs, volumes=scene_volumes,
              two_fluids=scene_two_fluids, **{"tail%d" % n: (lambda n=n: scene_tail(n)) for n in TAILS})


# ---- driving a world ---------------------------------------------------------------------------------------------------------
def populate(world, scene, forces=()):
    fh = []
    for f in scene["fluids"]:
        h = world.add_fluid(f["positions"], density0=f["density0"], velocities=f.get("velocities"), volumes=f.get("volumes"),
                            memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF))
        for kind, params in forces:
            world.push_force(h, kind, params)
        fh.append(h)
    bh = [world.add_boundary(b["positions"], velocities=b.get("velocities"), memberships=b.get("memberships", 1),
                             filter=b.get("filter", 0xFFFFFFFF), want_forces=b.get("want_forces", False))
          for b in scene["boundaries"]]
    return fh, bh


def _read(world, fh, bh):
    cat = lambda what: np.concatenate([world.debug(f, what) for f in fh])  # noqa: E731
    out = {w: cat(w) for w in ("density", "alpha", "divergence", "predicted_density", "velocity_change", "acceleration",
                               "num_fluid_contacts", "num_boundary_contacts")}
    pv = [world.read_fluid(f) for f in fh]
    out["P"] = np.concatenate([p for p, _ in pv])
    out["V"] = np.concatenate([v for _, v in pv])
    rb = [world.read_boundary(b) for b in bh]
    out["bvol"] = np.concatenate([v for v, _ in rb]) if bh else np.zeros(0, F)
    out["bforce"] = np.concatenate([f for _, f in rb]) if bh else np.zeros((0, 3), F)
    out["stats"] = world.stats()
    return out


def run(make_world, scene, iters, forces=(), first=None, **world_kw):
    """Step a fresh world once with force_iterations(*iters) (iters None: the solver's own loop), or twice when `first`
    gives the first step's iterations.  Returns the observables after the last step and, for two steps, those after the
    first.  world_kw goes to make_world (max_divergence_iter)."""
    w = make_world(**world_kw)
    fh, bh = populate(w, scene, forces)
    before = None
    if first is not None:
        w.force_iterations(*first)
        w.step(DT, ZERO_G)
        before = _read(w, fh, bh)
    if iters is not None:
        w.force_iterations(*iters)
    w.step(DT, ZERO_G)
    out = _read(w, fh, bh)
    if hasattr(w, "close"):
        w.close()
    return out, before


def passes_for(scene, P=None, kw=0, kg=0):
    """ref64.Passes of a scene (on positions P, default the scene's own)."""
    fl, bd = scene["fluids"], scene["boundaries"]
    pos = np.concatenate([f["positions"] for f in fl]).astype(F) if P is None else P
    fid = np.concatenate([np.full(len(f["positions"]), k) for k, f in enumerate(fl)])
    r = F(R)
    vdef = r * r * r * F(8.0 * 0.8)
    vol = np.concatenate([np.full(len(f["positions"]), vdef, F) if f.get("volumes") is None else np.asarray(f["volumes"], F)
                          for f in fl])
    rho0 = np.concatenate([np.full(len(f["positions"]), F(f["density0"]), F) for f in fl])
    mass = (vol * rho0).astype(F)
    bp = np.concatenate([b["positions"] for b in bd]).astype(F) if bd else np.zeros((0, 3), F)
    bid = np.concatenate([np.full(len(b["positions"]), k) for k, b in enumerate(bd)]) if bd else np.zeros(0, int)
    fm = np.array([f.get("memberships", 1) for f in fl], np.int64)
    ff_ = np.array([f.get("filter", 0xFFFFFFFF) for f in fl], np.int64)
    bm = np.array([b.get("memberships", 1) for b in bd], np.int64)
    bf_ = np.array([b.get("filter", 0xFFFFFFFF) for b in bd], np.int64)

    def test(m1, f1, m2, f2):
        return ((m1 & f2) != 0) & ((m2 & f1) != 0)

    def allowed_ff(i, j):
        a, b = fid[i], fid[j]
        return (a == b) | test(fm[a], ff_[a], fm[b], ff_[b])

    def allowed_fb(i, j):
        a, b = fid[i], bid[j]
        return test(fm[a], ff_[a], bm[b], bf_[b])

    def allowed_bb(i, j):
        a, b = bid[i], bid[j]
        return (a == b) | test(bm[a], bf_[a], bm[b], bf_[b])

    h = F(r * F(2.0) * F(2.0))
    return ref64.Passes(h, pos, fid, rho0, mass, bp, bid, allowed_ff, allowed_fb, allowed_bb, kw=kw, kg=kg)


# ---- the checks ----------------------------------------------------------------------------------------------------------------
MUTANTS = ("drop_entries_32_35", "swap_vy_vz_odd", "gate_at_21", "normals_rho_i", "boundary_mass_fluid0_rho0",
           "no_kappa_gate", "drop_last_boundary", "bforce_no_inv_dt", "artificial_no_vr_gate")


class Checks:
    """Runs the stages of one scene on one world kind and keeps the worst |err| / bound per pass.  `mutant` applies one
    plausible kernel bug to the reference instead (a bound that passes the mutant too is too loose)."""

    def __init__(self, make_world, scene, kw=0, kg=0, mutant=None):
        self.make_world, self.scene, self.mutant = make_world, scene, mutant
        self.ps = passes_for(scene, kw=kw, kg=kg)
        self.worst, self.excluded = {}, {}
        ps = self.ps
        self.ff, self.fb = ps.ff, ps.fb
        if mutant == "drop_entries_32_35":
            rk = ps.ff.rank()
            self.ff = ps.ff.subset(~((rk >= 32) & (rk < 36)))
        elif mutant == "drop_last_boundary":
            last = np.r_[ps.fb.i[1:] != ps.fb.i[:-1], True] if len(ps.fb.i) else np.zeros(0, bool)
            self.fb = ps.fb.subset(~last)
        self.rho0_b = np.full(ps.N, ps.rho0[0]) if mutant == "boundary_mass_fluid0_rho0" else None
        self.min_nb = 21 if mutant == "gate_at_21" else ref64.MIN_NEIGHBORS
        bd = scene["boundaries"]
        self.want = np.concatenate([np.full(len(b["positions"]), bool(b.get("want_forces", False))) for b in bd]) if bd else np.zeros(0, bool)

    def record_boundary(self, name, gpu, ref, ps=None):
        """Boundary forces of the boundaries that want them, per boundary particle; a boundary particle in contact with
        a pair at the gradient's zero threshold is excluded like a fluid one."""
        ps = ps or self.ps
        if not self.want.any():
            return
        r = ref64.ratio(gpu, ref, C_PASS["boundary_force"]).max(axis=1)
        t = ref64.grad_threshold(ps.kg, ps.h)
        ex = np.zeros(len(self.want), bool)
        ex[ps.fb.j[np.abs(ps.fb.d2 - t) <= 8 * ref64.U * t]] = True
        r = np.where(ex | ~self.want, 0.0, r)
        self.worst[name] = max(self.worst.get(name, 0.0), float(r.max()))
        self.excluded[name] = self.excluded.get(name, 0) + int((ex & self.want).sum())

    def record(self, name, gpu, ref, c_pass, exclude=None):
        r = ref64.ratio(gpu, ref, c_pass)
        if r.ndim == 2:
            r = r.max(axis=1)
        ex = self.ps.ambiguous() if exclude is None else exclude | self.ps.ambiguous()
        r = np.where(ex, 0.0, r)
        self.worst[name] = max(self.worst.get(name, 0.0), float(r.max()) if len(r) else 0.0)
        self.excluded[name] = self.excluded.get(name, 0) + int(ex.sum())
        return r

    def _vj(self, vs, pr):
        vj = np.asarray(vs, F)[pr.j].copy()
        if self.mutant == "swap_vy_vz_odd":
            odd = (pr.rank() & 1) == 1
            vj[odd] = vj[odd][:, [0, 2, 1]]
        return vj

    def stages(self):
        ps, sc = self.ps, self.scene
        o00, _ = run(self.make_world, sc, (0, 0))
        nf, nb = o00["num_fluid_contacts"].astype(np.int64), o00["num_boundary_contacts"].astype(np.int64)
        self.nf, self.nb = nf, nb
        cnt = np.where((nf == np.bincount(self.ff.i, minlength=ps.N)) & (nb == np.bincount(self.fb.i, minlength=ps.N)), 0.0, np.inf)
        self.worst["counts"] = float(cnt.max()) if len(cnt) else 0.0
        bvol = o00["bvol"]
        if len(bvol):
            sref = ps.boundary_volume_sum()
            r = ref64.ratio(1.0 / bvol.astype(np.float64), sref, C_PASS["boundary_volume"])
            self.worst["boundary_volume"] = float(r.max())
        kw = dict(ff=self.ff, fb=self.fb, rho0_b=self.rho0_b)
        self.record("density", o00["density"], ps.density(bvol, **kw), C_PASS["density"])
        self._alpha(o00["alpha"], bvol)
        V0 = np.concatenate([f["velocities"] for f in sc["fluids"]]).astype(F)
        self.record("divergence_sweep", o00["divergence"],
                    ps.divergence(V0, bvol, vj=self._vj(V0, self.ff), min_neighbors=self.min_nb, **kw), C_PASS["divergence"])
        bvel = np.concatenate([b["velocities"] for b in sc["boundaries"]]).astype(F)
        vs = (o00["V"] + (o00["acceleration"] * F(DT)).astype(F)).astype(F)
        self.record("predicted", o00["predicted_density"],
                    ps.divergence(vs, bvol, predicted=True, bvel=bvel, dens=o00["density"], dt=DT, vj=self._vj(vs, self.ff), **kw),
                    C_PASS["predicted"])
        o10, _ = run(self.make_world, sc, (1, 0))
        kappa = (o00["divergence"] * o00["alpha"]).astype(F)
        self.record("update", o10["V"], ps.update(kappa, bvol, V0, **kw), C_PASS["update"])
        self.record("divergence_eval", o10["divergence"],
                    ps.divergence(o10["V"], bvol, vj=self._vj(o10["V"], self.ff), min_neighbors=self.min_nb, **kw),
                    C_PASS["divergence"])
        o11, _ = run(self.make_world, sc, (1, 1))
        rho0 = ps.rho0.astype(F)
        kraw = ((o10["predicted_density"] - rho0).astype(F) * o10["alpha"]).astype(F)
        kp = np.maximum(kraw, F(0))
        inv_dt = F(1.0) / F(DT)
        vc0 = (o11["acceleration"] * F(DT)).astype(F)
        kb = kraw if self.mutant == "no_kappa_gate" else None
        self.record("pressure_update", o11["velocity_change"],
                    ps.update(kp, bvol, vc0, pressure=True, inv_dt=inv_dt, kappa_b=kb, **kw), C_PASS["update"])
        # boundary forces: the divergence update of the first step scales them by the previous inv_dt, 0; the pressure
        # update then adds (k_i vol_b rho0 inv_dt g) inv_dt m_i x_ib
        nb = len(self.want)
        self.record_boundary("boundary_force_first_step", o10["bforce"], ref64.Ref(np.zeros((nb, 3)), np.zeros((nb, 3)),
                                                                                   np.zeros((nb, 3)), np.zeros(nb)))
        self.record_boundary("boundary_force_pressure", o11["bforce"],
                             ps.pressure_boundary_force(kp, bvol, inv_dt, scale_m_inv_dt=self.mutant != "bforce_no_inv_dt"))
        return o00

    def _alpha(self, alpha, bvol):
        ref = self.ps.den(bvol, rho0_b=self.rho0_b)
        b = ref.bound(0)
        amb = np.abs(ref.value - 1e-5) <= b
        with np.errstate(divide="ignore", invalid="ignore"):
            den_gpu = np.where(alpha > 0, 1.0 / alpha.astype(np.float64), 0.0)
        # alpha = 0 <=> den <= 1e-5; otherwise 1 / alpha is den up to one more rounding of each reciprocal
            r = np.where(alpha > 0, np.abs(den_gpu - ref.value) / (b + 2 * ref64.U * np.abs(ref.value)),
                         np.where(ref.value <= 1e-5, 0.0, np.inf))
        r = np.where(amb | self.ps.ambiguous(), 0.0, r)
        self.worst["alpha"] = float(r.max()) if len(r) else 0.0
        self.excluded["alpha"] = int((amb | self.ps.ambiguous()).sum())

    def akinci(self, adhesion=0.0, gamma=1.0):
        """Unfused (0, 0); for a single uniform-mass fluid without adhesion, fused (1, 0) (force in the evaluation after the
        normals-carrying update); and the solver's own loop held to max_divergence_iter = 1, which ends on that update
        (force from k_akinci_force_u on its normals).  The acceleration is the force (gravity 0), on the stage's densities;
        with adhesion, the boundaries that want forces get -m_i times its boundary term."""
        from salva_b200 import scenes
        ps, sc = self.ps, self.scene
        forces = [scenes.akinci2013_surface_tension(gamma, adhesion)]
        for it, name, kw in (((0, 0), "akinci_unfused", {}), ((1, 0), "akinci_after_update", {}),
                             (None, "akinci_update_last", dict(max_divergence_iter=1))):
            o, _ = run(self.make_world, sc, it, forces, **kw)
            if it is None:
                assert o["stats"]["n_divergence_iter"] == 1 and o["stats"]["n_divergence_eval"] == 1
            if adhesion != 0 and it is not None:   # the free-running pressure loop adds its own boundary forces
                self.record_boundary("boundary_force_adhesion", o["bforce"], ps.adhesion_boundary_force(adhesion, o["bvol"]))
            rho_j = o["density"][self.ps.ff.i] if self.mutant == "normals_rho_i" else None
            ref = ps.akinci(o["density"], gamma, adhesion, o["bvol"], rho_j=rho_j, ff=self.ff, fb=self.fb)
            acc = o["acceleration"]
            assert np.isfinite(acc).all(), "%s: non-finite accelerations at %s" % (name, np.nonzero(~np.isfinite(acc).all(1))[0][:8])
            self.record(name, acc, ref, C_PASS["akinci"])

    def xsph(self, cf=0.5, cb=0.0):
        from salva_b200 import scenes
        sc = self.scene
        forces = [scenes.xsph_viscosity(cf, cb)]
        bvel = np.concatenate([b["velocities"] for b in sc["boundaries"]]).astype(F)
        for it, name in (((1, 0), "xsph_after_update"), ((0, 0), "xsph_separate")):
            o2, o1 = run(self.make_world, sc, it, forces, first=(1, 0))
            ps1 = passes_for(sc, P=o1["P"], kw=self.ps.kw, kg=self.ps.kg)
            assert np.array_equal(o2["num_fluid_contacts"], np.bincount(ps1.ff.i, minlength=ps1.N))
            ref = ps1.xsph(o2["V"], o2["density"], cf, cb, F(1.0) / F(DT), bvel, o2["bvol"])
            r = ref64.ratio(o2["acceleration"], ref, C_PASS["xsph"]).max(axis=1)
            r = np.where(ps1.ambiguous(), 0.0, r)
            self.worst[name] = max(self.worst.get(name, 0.0), float(r.max()))
            self.excluded[name] = self.excluded.get(name, 0) + int(ps1.ambiguous().sum())
            if it == (0, 0) and cb != 0:   # no update on step 2: the forces are XSPH's alone
                self.record_boundary("boundary_force_xsph", o2["bforce"],
                                     ps1.xsph_boundary_force(o2["V"], o2["density"], cb, F(1.0) / F(DT), bvel, o2["bvol"]), ps=ps1)

    def artificial(self, cf=1.0, cb=0.0, alpha=1.0, beta=0.0, cs=10.0):
        """ArtificialViscosity on the first step, with no update (0, 0) and after one (1, 0): it does not depend on dt, so
        the acceleration is its sum over the velocities the loop left and the step's densities.  Its boundary force is the
        running sum of the particle's boundary term (artificial_viscosity.rs:117), which depends on the order of the
        contact list, so it is not compared here."""
        from salva_b200 import scenes
        sc = self.scene
        forces = [scenes.artificial_viscosity(cf, cb, alpha, beta, cs)]
        bvel = np.concatenate([b["velocities"] for b in sc["boundaries"]]).astype(F)
        for it, name in (((0, 0), "artificial_no_update"), ((1, 0), "artificial_after_update")):
            o, _ = run(self.make_world, sc, it, forces)
            ref, amb = self.ps.artificial(o["V"], o["density"], cf, cb, alpha, beta, cs, bvel, o["bvol"],
                                          vr_gate=self.mutant != "artificial_no_vr_gate")
            assert amb.mean() <= 0.02, "%s: %d of %d particles at the v_r < 0 decision" % (name, amb.sum(), len(amb))
            self.record(name, o["acceleration"], ref, C_PASS["artificial"], exclude=amb)

    def flagged(self):
        return {k: v for k, v in self.worst.items() if not v <= 1.0}
