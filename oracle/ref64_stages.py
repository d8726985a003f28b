"""Feed each DFSPH gather pass its own inputs and check its output against oracle/ref64.py, particle by particle (the IISPH
passes: Checks.iisph_stages; the WCSPH, He2014, DFSPHViscosity and Becker2009 plugins: Checks.wcsph, .he2014, .viscosity,
.becker).

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


def light(scene):
    """The scene with every rest density divided by 1000.  DFSPHViscosity's matrix scales as 1 / rho0: at water's density
    its determinant lies below the 1e-6 gate almost everywhere and beta is 0; here it lies above."""
    out = dict(scene, fluids=[dict(f, density0=f["density0"] / 1000.0) for f in scene["fluids"]])
    return out


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


IISPH_SCRATCH = ("pressure", "dii", "aii", "dij_pjl")
HE2014_SCRATCH = ("he2014_color", "he2014_gradc")
VISC_SCRATCH = ("visc_beta", "visc_target")
EL_SCRATCH = ("el_volume0", "el_rotation", "el_grad_tr", "el_stress")


def deform(P, fid, angle, seed):
    """Each fluid's positions rotated by `angle` degrees about a tilted axis through its centre, stretched by a few percent
    along x and compressed along y, plus jitter of 0.2 % of the particle radius."""
    rng = np.random.default_rng(seed)
    ax = np.array([0.3, 1.0, 0.2]) / np.linalg.norm([0.3, 1.0, 0.2])
    t = np.radians(angle)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    rot = np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K
    M = rot @ np.diag([1.03, 0.98, 1.01])
    out = np.asarray(P, np.float64).copy()
    for k in np.unique(fid):
        sel = fid == k
        c = out[sel].mean(axis=0)
        out[sel] = c + (out[sel] - c) @ M.T
    return (out + rng.normal(0, 0.002 * R, out.shape)).astype(F)


def _read(world, fh, bh, extra=()):
    cat = lambda what: np.concatenate([world.debug(f, what) for f in fh])  # noqa: E731
    out = {w: cat(w) for w in ("density", "alpha", "divergence", "predicted_density", "velocity_change", "acceleration",
                               "num_fluid_contacts", "num_boundary_contacts") + tuple(extra)}
    pv = [world.read_fluid(f) for f in fh]
    out["P"] = np.concatenate([p for p, _ in pv])
    out["V"] = np.concatenate([v for _, v in pv])
    rb = [world.read_boundary(b) for b in bh]
    out["bvol"] = np.concatenate([v for v, _ in rb]) if bh else np.zeros(0, F)
    out["bforce"] = np.concatenate([f for _, f in rb]) if bh else np.zeros((0, 3), F)
    out["stats"] = world.stats()
    return out


def run(make_world, scene, iters, forces=(), first=None, extra=(), **world_kw):
    """Step a fresh world once with force_iterations(*iters) (iters None: the solver's own loop), or twice when `first`
    gives the first step's iterations.  Returns the observables after the last step and, for two steps, those after the
    first.  extra: further debug selectors to read (IISPH_SCRATCH); world_kw goes to make_world (max_divergence_iter,
    min_pressure_iter, max_pressure_iter)."""
    w = make_world(**world_kw)
    fh, bh = populate(w, scene, forces)
    before = None
    if first is not None:
        w.force_iterations(*first)
        w.step(DT, ZERO_G)
        before = _read(w, fh, bh, extra)
    if iters is not None:
        w.force_iterations(*iters)
    w.step(DT, ZERO_G)
    out = _read(w, fh, bh, extra)
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
           "no_kappa_gate", "drop_last_boundary", "bforce_no_inv_dt", "artificial_no_vr_gate",
           # IISPH
           "dji_mass_j", "s_without_dii_p", "dij_prho_i", "next_p_no_boundary", "no_relaxation", "velocity_prho_i_twice",
           "no_warm_start", "error_counts_clamped", "iisph_bforce_no_mass",
           # surface tension plugins
           "wcsph_inverted_mass_ratio", "he2014_colors_no_boundary", "he2014_gradc_by_cj", "he2014_gradc_i_twice",
           "he2014_reaction_sign",
           # Becker2009 elasticity
           "el_volume_once", "el_r_i_for_r_j", "el_g_i_for_g_j", "el_rest_lists_recaptured",
           "el_recapture_no_old_volumes", "el_second_fluid_no_offset",
           # DFSPHViscosity
           "visc_precondition_columns", "visc_target_no_scale", "visc_vv_no_adt", "visc_u_j_beta_i")


class Checks:
    """Runs the stages of one scene on one world kind and keeps the worst |err| / bound per pass.  `mutant` applies one
    plausible kernel bug to the reference instead (a bound that passes the mutant too is too loose)."""

    def __init__(self, make_world, scene, kw=0, kg=0, mutant=None):
        self.make_world, self.scene, self.mutant = make_world, scene, mutant
        self.ps = passes_for(scene, kw=kw, kg=kg)
        self.worst, self.excluded, self.clamp = {}, {}, {}
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

    def record(self, name, gpu, ref, c_pass, exclude=None, ps=None, ambiguous=True):
        """ambiguous = False: the pass does not run on ps's contacts (Becker's rest contacts), so ps's pairs at the
        gradient's zero threshold do not exclude anything."""
        ps = ps or self.ps
        r = ref64.ratio(gpu, ref, c_pass)
        if r.ndim == 2:
            r = r.max(axis=1)
        amb = ps.ambiguous() if ambiguous else np.zeros(len(r), bool)
        ex = amb if exclude is None else exclude | amb
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

    def _first_step_lists(self, o00, alpha=True):
        """Counts, boundary volumes, rho and (alpha) alpha of a first step (the neighbour search and the density pass)."""
        ps = self.ps
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
        if alpha:
            self._alpha(o00["alpha"], bvol)
        return bvol, kw

    def stages(self):
        ps, sc = self.ps, self.scene
        o00, _ = run(self.make_world, sc, (0, 0))
        bvol, kw = self._first_step_lists(o00)
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

    def iisph_stages(self, omega=0.5, alpha=True):
        """The IISPH passes, on a world made with the IISPH solver (make_world takes min_pressure_iter and
        max_pressure_iter).  Gravity 0 and no forces: acc = 0, so v* = V0.  alpha: the world computes alpha under IISPH too
        (the engine's density pass does; the CPU oracle's IISPH, like the reference's, does not).
          (0, 0)  counts, boundary volumes, rho and alpha (the density pass), dii, aii (fed dii as read back), the
                  predicted density, p = 0 and V = V0;
          (0, 1)  p_1 (dij_pjl = 0 and s = 0 here; fed the reference's predicted density, so it sees that pass's
                  boundary term too), then V and the boundary forces on p_1;
          (0, 2)  dij_pjl fed p_1, and p_2 fed p_1 and this run's aii, dii, dij_pjl: s_j, d_ji p_i and the boundary term;
          error   the free-running loop held to k = 1, 2 iterations: last_density_error;
          warm    step 1 with (0, 2), step 2 with (0, 1) on contacts re-derived on P1: dij_pjl and p fed 0.5 p_2 of each
                  particle, which checks that pressures ride the step's counting sort.
        The |aii| > 1e-9 gate is an exact decision on the float32 aii the kernel reads, so it needs no exclusion.  A
        nonzero |aii| <= 1e-9 needs a particle with a few contacts near the support's edge, whose density is about a
        quarter of rho0 and whose pressure is clamped to 0 whether or not the gate fires; so the gate shows only at
        aii = 0, which the lone particle of tail1 reaches."""
        ps, sc, m = self.ps, self.scene, self.mutant
        X = IISPH_SCRATCH
        o0, _ = run(self.make_world, sc, (0, 0), extra=X)
        bvol, kw = self._first_step_lists(o0, alpha)
        dens = o0["density"]
        V0 = np.concatenate([f["velocities"] for f in sc["fluids"]]).astype(F)
        bvel = np.concatenate([b["velocities"] for b in sc["boundaries"]]).astype(F)
        pred = ps.divergence(V0, bvol, predicted=True, bvel=bvel, dens=dens, dt=DT, **kw)
        self.record("predicted", o0["predicted_density"], pred, C_PASS["predicted"])
        self.record("dii", o0["dii"], ps.iisph_dii(dens, bvol, DT, **kw), C_PASS["iisph_dii"])
        dji_mass = ps.mass[self.ff.j] if m == "dji_mass_j" else None
        self.record("aii", o0["aii"], ps.iisph_aii(dens, o0["dii"], bvol, DT, dji_mass=dji_mass, **kw), C_PASS["iisph_aii"])
        self.worst["pressure_0"] = 0.0 if not o0["pressure"].any() and np.array_equal(o0["V"], V0) else np.inf

        pk = dict(dji_mass=dji_mass, s_dii_p=m != "s_without_dii_p", boundary=m != "next_p_no_boundary", **kw)
        relax = m != "no_relaxation"
        o1, _ = run(self.make_world, sc, (0, 1), extra=X)
        ref, raw = ps.iisph_next_pressure(o1["density"], pred.value, o0["pressure"], o1["aii"], o1["dii"], o1["dij_pjl"], bvol,
                                          DT, omega, pred_err=pred.bound(C_PASS["predicted"]), relax=relax, **pk)
        self._pressure("pressure_1", o1["pressure"], ref, raw)
        p1 = o1["pressure"]
        self.record("velocity", o1["V"], ps.iisph_velocity(dens, p1, V0, bvol, DT, prho_i_twice=m == "velocity_prho_i_twice", **kw),
                    C_PASS["iisph_velocity"])
        self.record_boundary("boundary_force_iisph", o1["bforce"],
                             ps.iisph_boundary_force(dens, p1, bvol, rho0_b=self.rho0_b, with_mass=m != "iisph_bforce_no_mass"))

        o2, _ = run(self.make_world, sc, (0, 2), extra=X)
        self.record("dij_pjl", o2["dij_pjl"], ps.iisph_dij_pjl(dens, p1, DT, prho_i=m == "dij_prho_i", ff=self.ff),
                    C_PASS["iisph_dij_pjl"])
        ref, raw = ps.iisph_next_pressure(dens, o2["predicted_density"], p1, o2["aii"], o2["dii"], o2["dij_pjl"], bvol, DT, omega,
                                          relax=relax, **pk)
        self._pressure("pressure_2", o2["pressure"], ref, raw)

        for k, p_prev in ((1, o0["pressure"]), (2, p1)):
            o, _ = run(self.make_world, sc, None, extra=X, min_pressure_iter=k, max_pressure_iter=k)
            assert o["stats"]["n_pressure_iter"] == k, o["stats"]
            v, b, amb = ps.iisph_density_error(o["density"], o["predicted_density"], p_prev, o["aii"], o["dii"], o["dij_pjl"],
                                               o["bvol"], DT, omega, C_PASS["iisph_pressure"],
                                               count_clamped=m == "error_counts_clamped", relax=relax, **pk)
            err = abs(float(o["stats"]["last_density_error"]) - v)
            self.worst["density_error"] = max(self.worst.get("density_error", 0.0), err / b if b > 0 else (0.0 if err == 0 else np.inf))
            self.excluded["density_error"] = self.excluded.get("density_error", 0) + amb

        o2w, o1w = run(self.make_world, sc, (0, 1), first=(0, 2), extra=X)
        ps1 = passes_for(sc, P=o1w["P"], kw=ps.kw, kg=ps.kg)
        assert np.array_equal(o2w["num_fluid_contacts"], ps1.nf) and np.array_equal(o2w["num_boundary_contacts"], ps1.nb)
        p_ws = o1w["pressure"] if m == "no_warm_start" else (o1w["pressure"] * F(0.5)).astype(F)
        self.record("dij_pjl_warm", o2w["dij_pjl"], ps1.iisph_dij_pjl(o2w["density"], p_ws, DT), C_PASS["iisph_dij_pjl"], ps=ps1)
        ref, raw = ps1.iisph_next_pressure(o2w["density"], o2w["predicted_density"], p_ws, o2w["aii"], o2w["dii"], o2w["dij_pjl"],
                                           o2w["bvol"], DT, omega)
        self._pressure("pressure_warm", o2w["pressure"], ref, raw, ps=ps1)
        self.moved_cells = int((np.floor(o1w["P"] / ps.h) != np.floor(ps.P / ps.h)).any(axis=1).sum())
        return o0

    def _pressure(self, name, gpu, ref, raw, ps=None):
        """A pressure pass: particles whose unclamped value lies within its bound of 0 are excluded (the clamp may go either
        way); the others are counted on each side of the clamp."""
        b = ref.bound(C_PASS["iisph_pressure"])
        amb = np.abs(np.nan_to_num(raw)) <= b
        amb &= ~np.isnan(raw)
        self.record(name, gpu, ref, C_PASS["iisph_pressure"], exclude=amb, ps=ps)
        side = self.clamp.setdefault(name, [0, 0])
        side[0] += int((np.nan_to_num(raw) < -b).sum())
        side[1] += int((np.nan_to_num(raw) > b).sum())

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

    def wcsph(self, cf=0.5):
        """WCSPHSurfaceTension on the first step with no update (0, 0): the acceleration is its fluid term.  Its boundary
        coefficient must be 0 (include/sph.h), so there is no boundary term."""
        from salva_b200 import scenes
        o, _ = run(self.make_world, self.scene, (0, 0), [scenes.wcsph_surface_tension(cf)])
        ref = self.ps.wcsph(cf, inverted_mass_ratio=self.mutant == "wcsph_inverted_mass_ratio")
        self.record("wcsph", o["acceleration"], ref, C_PASS["wcsph"])

    def he2014(self, cf=0.5, cb=0.3):
        """He2014SurfaceTension on the first step with no update (0, 0), each pass fed what its kernel read: the colours on
        the step's densities, gradc on the colours read back, the acceleration (the force: gravity 0) and the boundary
        reaction on gradc read back.  With cb = 0 the boundaries that want forces get none."""
        from salva_b200 import scenes
        ps, m = self.ps, self.mutant
        o, _ = run(self.make_world, self.scene, (0, 0), [scenes.he2014_surface_tension(cf, cb)], extra=HE2014_SCRATCH)
        dens, bvol = o["density"], o["bvol"]
        self.record("he2014_color", o["he2014_color"], ps.he2014_colors(dens, bvol, boundary=m != "he2014_colors_no_boundary"),
                    C_PASS["he2014_color"])
        self.record("he2014_gradc", o["he2014_gradc"],
                    ps.he2014_gradc(dens, o["he2014_color"], C_PASS["he2014_gradc"], divide_by_cj=m == "he2014_gradc_by_cj"), 0)
        tag = "fluid" if cb == 0 else "boundary" if cf == 0 else "both"
        self.record("he2014_force_" + tag, o["acceleration"],
                    ps.he2014_force(dens, o["he2014_gradc"], cf, cb, bvol, gradc_i_twice=m == "he2014_gradc_i_twice"), C_PASS["he2014_force"])
        if cb != 0:
            ref = ps.he2014_boundary_force(dens, o["he2014_gradc"], cb, bvol, sign=1.0 if m == "he2014_reaction_sign" else -1.0)
        else:
            nb = len(self.want)
            ref = ref64.Ref(np.zeros((nb, 3)), np.zeros((nb, 3)), np.zeros((nb, 3)), np.zeros(nb))
        self.record_boundary("boundary_force_he2014", o["bforce"], ref)

    def viscosity(self, visc=0.5, wcsph=0.0):
        """DFSPHViscosity.  Forces see the previous step's dt, 0 on the first step, so (as for XSPH) step 1 with (1, 0),
        then step 2 with (0, 0) on positions P1, the velocities V2 and the densities of step 2, once with
        max_viscosity_iter = 1 and once with 2 (max_viscosity_error = 0: no early break).  Each pass fed what its kernel
        read: beta (residual check), the target on vv = v + a dt, the acceleration after one update (rate on the same vv,
        beta and target read back) and after two (vv on the acceleration read back from the one-update run).  wcsph: a
        WCSPHSurfaceTension coefficient pushed before the viscosity, so that a != 0 in vv; its acceleration comes from a
        run with WCSPH alone."""
        from salva_b200 import scenes
        sc, m, kw = self.scene, self.mutant, dict(kw=self.ps.kw, kg=self.ps.kg)
        tag = "_after_wcsph" if wcsph else ""
        pre = [scenes.wcsph_surface_tension(wcsph)] if wcsph else []
        runs = {k: run(self.make_world, sc, (0, 0), pre + [scenes.dfsph_viscosity(visc, 1, k, 0.0)], first=(1, 0), extra=VISC_SCRATCH)
                for k in (1, 2)}
        o2, o1 = runs[1]
        ps1 = passes_for(sc, P=o1["P"], **kw)
        dens, V = o2["density"], o2["V"]
        a0 = run(self.make_world, sc, (0, 0), pre, first=(1, 0))[0]["acceleration"] if wcsph else np.zeros_like(V)
        ratio, viol, amb, zero = ps1.visc_beta(dens, o2["visc_beta"], C_PASS["visc_matrix"], by_column=m == "visc_precondition_columns")
        amb = amb | ps1.ambiguous()
        self.worst["visc_beta" + tag] = max(self.worst.get("visc_beta" + tag, 0.0), float(np.where(amb, 0.0, ratio).max()))
        self.worst["visc_beta_gate" + tag] = np.inf if viol else 0.0
        self.excluded["visc_beta" + tag] = self.excluded.get("visc_beta" + tag, 0) + int(amb.sum())
        self.visc_zero = getattr(self, "visc_zero", 0) + int(zero.sum())
        skip = m == "visc_vv_no_adt"
        scale = 1.0 if m == "visc_target_no_scale" else float(F(1.0) - F(visc))
        self.record("visc_target" + tag, o2["visc_target"], ps1.visc_rates(dens, V, a0, DT, scale, skip_adt=skip),
                    C_PASS["visc_rate"] + 1, ps=ps1)
        inv_dt = F(1.0) / F(DT)
        acc = a0
        for k in (1, 2):
            ok = runs[k][0]
            rate = ps1.visc_rates(dens, V, acc, DT, 1.0, skip_adt=skip)
            ref = ps1.visc_accel(dens, ok["visc_beta"], rate.value, rate.bound(C_PASS["visc_rate"]), ok["visc_target"], acc, inv_dt,
                                 beta_i_for_j=m == "visc_u_j_beta_i")
            self.record("visc_accel_%d%s" % (k, tag), ok["acceleration"], ref, C_PASS["visc_accel"], ps=ps1)
            acc = runs[1][0]["acceleration"]

    def becker(self, young=2.0e5, poisson=0.3, nonlinear=True, angle=40.0):
        """Becker2009Elasticity, every pass fed what its kernel read (rest volumes, rotations, grad_tr and stress read
        back), with no update (0, 0) so that the acceleration is the force:
          step 1  captures the rest pose (the step's positions and same-fluid contacts): the rest volumes; the rotation
                  within its bound of the polar rotation, which is I here; grad_tr, stress and force near 0;
          step 2  after write_fluid imposed a deformation of each fluid about its centre (a rotation by `angle` degrees
                  about a tilted axis, a few percent of strain and jitter): the current contacts differ from the rest
                  contacts, and rotation, grad_tr, stress and force are checked on the rest contacts;
          step 3  a further deformation (25 degrees): the rotation warm-started from step 2's;
          step 4  after appending particles to every fluid: the rest pose is captured again, with the old rest volumes
                  added to the new sums and the old rotations kept as warm starts (identity for the new particles)
                  (becker2009_elasticity.rs:84-113, Vec::resize)."""
        from salva_b200 import scenes
        sc, ps, m = self.scene, self.ps, self.mutant
        w = self.make_world()
        fh, bh = populate(w, sc, [scenes.becker2009_elasticity(young, poisson, nonlinear)])
        w.force_iterations(0, 0)
        Q = np.concatenate([f["positions"] for f in sc["fluids"]]).astype(F)
        same = lambda fid: (lambda i, j: fid[i] == fid[j])  # noqa: E731
        bk = ref64.Becker(ps.h, Q, ps.fid, ps.mass, young, poisson, nonlinear)
        tag = "nonlinear" if nonlinear else "linear"
        w.step(DT, ZERO_G)
        o = _read(w, fh, bh, EL_SCRATCH)
        self.record("el_volume", ps.mass / o["el_volume0"].astype(np.float64), bk.volume_sum(1.0 if m == "el_volume_once" else 2.0),
                    C_PASS["el_volume"], exclude=np.zeros(ps.N, bool), ambiguous=False)
        self._becker_step(bk, Q, o, np.tile(np.eye(3), (ps.N, 1, 1)), "el_rest_" + tag)
        R_prev = o["el_rotation"].reshape(ps.N, 3, 3).astype(np.float64)
        if m == "el_rest_lists_recaptured":
            P2 = deform(o["P"], ps.fid, angle, seed=29)
            bk = ref64.Becker(ps.h, Q, ps.fid, ps.mass, young, poisson, nonlinear, rest=ref64.contacts(P2, P2, ps.h, same(ps.fid), same=True))
        for name, ang, seed in (("el_deformed_", angle, 29), ("el_warm_", 25.0, 31)):
            P = deform(o["P"], ps.fid, ang, seed=seed)
            for k, f in enumerate(fh):
                w.write_fluid(f, positions=P[ps.fid == k])
            w.step(DT, ZERO_G)
            o = _read(w, fh, bh, EL_SCRATCH)
            self._becker_step(bk, P, o, R_prev, name + tag)
            R_prev = o["el_rotation"].reshape(ps.N, 3, 3).astype(np.float64)
            if name == "el_deformed_":   # rest contacts against the same-fluid contacts at P
                cur = ref64.contacts(P, P, ps.h, same(ps.fid), same=True)
                self.rest_differs = int((np.bincount(bk.rest.i, minlength=ps.N) != np.bincount(cur.i, minlength=ps.N)).sum())
        # re-capture: 7 particles appended to every fluid, near particles of it
        P, vol0 = o["P"], o["el_volume0"]
        vdef = F(R) * F(R) * F(R) * F(8.0 * 0.8)
        pos, fid, mass, old_vol, old_rot = [], [], [], [], []
        for k, f in enumerate(fh):
            sel = np.nonzero(ps.fid == k)[0]
            new = (P[sel[5:68:9]] + np.array([0.4, 0.1, 0.2], F) * F(R)).astype(F)
            w.append_particles(f, new)
            pos += [P[sel], new]
            fid += [np.full(len(sel) + len(new), k)]
            mass += [ps.mass[sel], np.full(len(new), F(vdef * F(sc["fluids"][k]["density0"])), F)]   # appended: default volume
            old_vol += [vol0[sel], np.zeros(len(new))]
            old_rot += [R_prev[sel], np.tile(np.eye(3), (len(new), 1, 1))]
        Q4, fid4, mass4 = np.concatenate(pos).astype(F), np.concatenate(fid), np.concatenate(mass).astype(F)
        w.step(DT, ZERO_G)
        o = _read(w, fh, bh, EL_SCRATCH)
        bk4 = ref64.Becker(ps.h, Q4, fid4, mass4, young, poisson, nonlinear)
        old = np.zeros(len(Q4)) if m == "el_recapture_no_old_volumes" else np.concatenate(old_vol)
        self.record("el_recaptured_volume", mass4 / o["el_volume0"].astype(np.float64),
                    bk4.volume_sum(2.0, old=old), C_PASS["el_volume"],
                    exclude=np.zeros(len(Q4), bool), ambiguous=False)
        self._becker_step(bk4, Q4, o, np.concatenate(old_rot), "el_recaptured_" + tag)
        if hasattr(w, "close"):
            w.close()

    def _becker_step(self, bk, P, o, R_prev, name):
        N, m = bk.N, self.mutant
        R = o["el_rotation"].reshape(N, 3, 3).astype(np.float64)
        G = o["el_grad_tr"].reshape(N, 3, 3)
        if m == "el_second_fluid_no_offset" and bk.fid.max() > 0:   # the second fluid reads the first one's positions
            P = np.asarray(P, F).copy()
            sel = np.nonzero(bk.fid == 1)[0]
            P[sel] = P[np.nonzero(bk.fid == 0)[0][:len(sel)]]
        none = np.zeros(N, bool)
        r, ortho, ex, Rref, iters = bk.rotation(P, R, R_prev, C_PASS["el_apq"])
        # the scenes' edges: how far the float64 run turned from its warm start, in how many iterations, and that it ends
        # on the polar rotation (no other stationary point of the iteration)
        ok = ~ex
        turn = np.degrees(np.arccos(np.clip((np.einsum("nij,nij->n", R_prev, Rref) - 1) / 2, -1, 1)))
        self.el_turn = max(getattr(self, "el_turn", 0.0), float(turn[ok].min()) if ok.any() else 0.0)
        self.el_iterations = max(getattr(self, "el_iterations", 0), int(iters[ok].max()) if ok.any() else 0)
        gap = np.abs(Rref - bk.polar(bk.apq(P, C_PASS["el_apq"])[0])).max(axis=(1, 2))
        self.el_polar_gap = max(getattr(self, "el_polar_gap", 0.0), float(gap[ok].max()) if ok.any() else 0.0)
        self.worst[name + "_rotation"] = max(self.worst.get(name + "_rotation", 0.0), float(r.max()))
        self.excluded[name + "_rotation"] = self.excluded.get(name + "_rotation", 0) + int(ex.sum())
        self.worst[name + "_orthonormal"] = max(self.worst.get(name + "_orthonormal", 0.0), float(ortho.max()))
        kw = dict(exclude=none, ambiguous=False)
        self.record(name + "_grad_tr", G.reshape(N, 9), bk.grad_tr(P, R, o["el_volume0"]), C_PASS["el_grad_tr"], **kw)
        self.record(name + "_stress", o["el_stress"], bk.stress(G), ref64.C_EL_STRESS, **kw)
        self.record(name + "_force", o["acceleration"],
                    bk.force(o["el_stress"], G, R, o["el_volume0"], r_i_for_r_j=m == "el_r_i_for_r_j",
                             g_i_for_g_j=m == "el_g_i_for_g_j"), C_PASS["el_force"], **kw)

    def flagged(self):
        return {k: v for k, v in self.worst.items() if not v <= 1.0}
