"""Vorticity confinement (include/sph.h SPH_FORCE_VORTICITY_CONFINEMENT, DESIGN.md section 18): its three passes restated in
float64 over ref64.Passes, with the scale each float32 evaluation's error is measured against; a float32 CPU twin of the
force for OracleWorld; and Checks.vorticity, which replays a world and feeds each pass what its kernel read.

TEST INFRASTRUCTURE ONLY.  The force has no reference counterpart; the rule is the header's:
  omega_i = sum_j V_j grad W_ij x (v_j - v_i)
  eta_i   = sum_j V_j (|omega_j| - |omega_i|) grad W_ij
  a_i    += eps (N_i x omega_i),  N_i = eta_i / |eta_i| (0 where eta_i = 0)
over the contacts of i's own fluid (self included), V_j = m_j / rho_j.  omega and eta cancel in the interior, so each is bounded
per component (the Ref's A = 0, K the whole bound), as ref64.Passes.he2014_gradc is.
"""
import numpy as np

from . import ref64
from . import ref64_stages as S
from .oracle import OracleWorld
from .ref64 import C_NORM, U, F, Ref

KIND = 7                       # SPH_FORCE_VORTICITY_CONFINEMENT
SCRATCH = ("vorticity", "vorticity_eta")
C_PASS = dict(
    # omega: V_j = m_j / rho_j 1, g V_j 1, v_j - v_i 1, x_ij 1, the cross product's two products and difference 3, fma 1,
    # g 6.2; margin 1.8
    vorticity_omega=C_NORM + 16,
    # eta: V_j 1, g V_j 1, |omega_j| - |omega_i| 1 and each norm's squares, sums and square root 4 (carried in A through
    # |omega_j| + |omega_i|), * 1, x_ij 1, fma 1, g 6.2; margin 1.8
    vorticity_eta=C_NORM + 18,
    # force, from the float32 omega and eta: |eta| 4, eta / |eta| 1, the cross product 3, * eps 1, acc + 1; margin 2
    vorticity_force=12,
)


def _f64(a):
    return np.asarray(a, F).astype(np.float64)


def _cross_abs(a, b):
    """The cross product's absolute evaluation |a_y||b_z| + |a_z||b_y|, ... per row."""
    a, b = np.abs(a), np.abs(b)
    return np.stack([a[:, 1] * b[:, 2] + a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] + a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] + a[:, 1] * b[:, 0]], 1)


# ---- the float64 passes ----------------------------------------------------------------------------------------------------
def omega(ps, vel, dens, c_pass, v_i_minus_v_j=False, rho_i=False, any_fluid=False, bvel=None, bvol=None):
    """omega_i = sum_j V_j grad W_ij x (v_j - v_i) on ref64.Passes ps.  Mutants: v_i_minus_v_j (the sign of omega), rho_i
    (1 / rho_i for 1 / rho_j), any_fluid (other fluids' neighbours too), bvel / bvol given (boundary contacts too, V_b = vol_b)."""
    N, v, rho = ps.N, _f64(vel), _f64(dens)
    prs = [(ps.ff if any_fluid else ps._same(), v, None)]
    if bvel is not None:
        prs.append((ps.fb, _f64(bvel), _f64(bvol)))
    val, e, n = np.zeros((N, 3)), np.zeros((N, 3)), np.zeros(N)
    for pr, vj, bv in prs:
        g, _, ge = ps._g(pr)
        vol = bv[pr.j] if bv is not None else ps.mass[pr.j] / rho[pr.i if rho_i else pr.j]
        u = vj[pr.j] - v[pr.i]
        if v_i_minus_v_j:
            u = -u
        cA = _cross_abs(pr.x, u)
        nk = ps._n(pr).astype(np.float64)
        val += ref64._sum(N, pr.i, (vol * g)[:, None] * np.cross(pr.x, u))
        e += (nk + c_pass)[:, None] * U * ref64._sum(N, pr.i, np.abs(vol * g)[:, None] * cA) + ref64._sum(N, pr.i, (np.abs(vol) * ge)[:, None] * cA)
        n += nk
    return Ref(val, np.zeros((N, 3)), e, n)


def eta(ps, dens, om, c_pass, plain_sum=False):
    """eta_i = sum_j V_j (|omega_j| - |omega_i|) grad W_ij over the float32 omega the kernel read.  plain_sum (mutant):
    sum_j V_j |omega_j| grad W_ij."""
    sf, N = ps._same(), ps.N
    wn = np.sqrt((_f64(om) ** 2).sum(1))
    wi = 0.0 if plain_sum else wn[sf.i]
    Vj = ps.mass[sf.j] / _f64(dens)[sf.j]
    a, aA, aK = ps._grad_terms(sf, Vj * (wn[sf.j] - wi), Vj * (wn[sf.j] + wi))
    n = ps._n(sf).astype(np.float64)
    e = (n + c_pass)[:, None] * U * ref64._sum(N, sf.i, aA) + ref64._sum(N, sf.i, aK)
    return Ref(ref64._sum(N, sf.i, a), np.zeros((N, 3)), e, n)


def ill_conditioned(eta_ref):
    """Particles whose eta bound reaches |eta| / 4: N = eta / |eta| is ill-conditioned there."""
    b = np.sqrt((eta_ref.bound(0) ** 2).sum(1))
    return b >= 0.25 * np.sqrt((eta_ref.value ** 2).sum(1))


def force(om, et, eps, omega_x_n=False, unnormalised=False):
    """eps (N x omega) from the float32 omega and eta the kernel read: a Ref whose A is the cross product's absolute
    evaluation.  Mutants: omega_x_n (omega x N), unnormalised (eta for N)."""
    w, e = _f64(om), _f64(et)
    en = np.sqrt((e * e).sum(1))
    nv = e if unnormalised else np.where(en[:, None] > 0, e / np.where(en > 0, en, 1.0)[:, None], 0.0)
    eps = float(F(eps))
    val = eps * (np.cross(w, nv) if omega_x_n else np.cross(nv, w))
    N = len(w)
    return Ref(val, eps * _cross_abs(nv, w), np.zeros((N, 3)), np.zeros(N))


# ---- the float32 CPU twin ----------------------------------------------------------------------------------------------------
class OracleVorticityWorld(OracleWorld):
    """OracleWorld with SPH_FORCE_VORTICITY_CONFINEMENT: the force runs as a host force at its slot in push order, on the
    positions, velocities and densities the oracle's forces read there, in float32 over the fluid's own contacts (the float32
    test (dx*dx + dy*dy) + dz*dz <= h*h, self included) with the solver's gradient kernel.  debug() reads omega and eta under
    the plugin-scratch rule: refused (AssertionError, as OracleWorld refuses) before the first solve and after particles were
    appended or deleted."""

    def __init__(self, particle_radius, smoothing_factor=2.0, kernel_gradient=0, **kw):
        super().__init__(particle_radius, smoothing_factor, kernel_gradient=kernel_gradient, **kw)
        self._kg = kernel_gradient
        self._mass, self._vort = {}, {}

    def add_fluid(self, positions, density0=1000.0, velocities=None, volumes=None, **kw):
        h = super().add_fluid(positions, density0=density0, velocities=velocities, volumes=volumes, **kw)
        n = len(np.asarray(positions).reshape(-1, 3))
        vol = np.full(n, self._default_volume(), F) if volumes is None else np.asarray(volumes, F)
        self._mass[h] = (vol * F(density0)).astype(F), F(density0)
        return h

    def _default_volume(self):
        r = F(self.particle_radius)
        return r * r * r * F(8.0 * 0.8)

    def push_force(self, fluid, kind, params):
        if kind != KIND:
            return super().push_force(fluid, kind, params)
        eps = F(params[0])
        assert np.isfinite(eps) and eps > 0, "vorticity confinement: eps must be finite and > 0"
        self.push_host_force(fluid, lambda dt, inv_dt, h, P, V, dens, acc: self._solve(fluid, eps, h, P, V, dens, acc))

    def append_particles(self, fluid, positions, velocities=None):
        super().append_particles(fluid, positions, velocities)
        m, rho0 = self._mass[fluid]
        n = len(np.asarray(positions).reshape(-1, 3))
        self._mass[fluid] = np.concatenate([m, np.full(n, F(self._default_volume() * rho0), F)]), rho0
        self._vort.pop(fluid, None)

    def delete_particles(self, fluid, mask):
        super().delete_particles(fluid, mask)
        m, rho0 = self._mass[fluid]
        self._mass[fluid] = m[~np.asarray(mask, bool)], rho0   # the particles leave at the start of the next step, before forces
        self._vort.pop(fluid, None)

    def _solve(self, fluid, eps, h, P, V, dens, acc):
        P, V, dens = np.array(P, F), np.array(V, F), np.array(dens, F)
        m = self._mass[fluid][0]
        pr = ref64.contacts(P, P, float(h), lambda i, j: np.ones(len(i), bool), same=True)
        d = (P[pr.i] - P[pr.j]).astype(F)
        d2 = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F)
        g = ref64.kernel(self._kg, "g", np.sqrt(d2.astype(np.float64)), float(h))[0]
        g = np.where(d2 <= ref64.grad_threshold(self._kg, float(h)), 0.0, g).astype(F)
        c = (g * (m[pr.j] / dens[pr.j])).astype(F)
        u = (V[pr.j] - V[pr.i]).astype(F)
        cr = np.stack([d[:, 1] * u[:, 2] - d[:, 2] * u[:, 1], d[:, 2] * u[:, 0] - d[:, 0] * u[:, 2],
                       d[:, 0] * u[:, 1] - d[:, 1] * u[:, 0]], 1).astype(F)
        om = np.zeros((len(P), 3), F)
        np.add.at(om, pr.i, (c[:, None] * cr).astype(F))
        wn = np.sqrt((om[:, 0] * om[:, 0] + om[:, 1] * om[:, 1]) + om[:, 2] * om[:, 2]).astype(F)
        t = (c * (wn[pr.j] - wn[pr.i])).astype(F)
        et = np.zeros((len(P), 3), F)
        np.add.at(et, pr.i, (t[:, None] * d).astype(F))
        en = np.sqrt((et[:, 0] * et[:, 0] + et[:, 1] * et[:, 1]) + et[:, 2] * et[:, 2]).astype(F)
        nv = np.where(en[:, None] > 0, et / np.where(en > 0, en, F(1.0))[:, None], F(0.0)).astype(F)
        acc += eps * np.stack([nv[:, 1] * om[:, 2] - nv[:, 2] * om[:, 1], nv[:, 2] * om[:, 0] - nv[:, 0] * om[:, 2],
                               nv[:, 0] * om[:, 1] - nv[:, 1] * om[:, 0]], 1).astype(F)
        self._vort[fluid] = om, et

    def debug(self, fluid, what):
        if what not in SCRATCH:
            return super().debug(fluid, what)
        assert fluid in self._vort, "selector %s needs a vorticity confinement solved with the fluid's current particles" % what
        return self._vort[fluid][SCRATCH.index(what)].copy()


# ---- replaying a world ----------------------------------------------------------------------------------------------------------
class Checks(S.Checks):
    """ref64_stages.Checks with the vorticity confinement stage.  Mutants (applied to the reference): vort_v_i_minus_v_j,
    vort_rho_i, vort_other_fluids, vort_boundaries, vort_eta_plain_sum, vort_omega_x_n, vort_unnormalised."""

    def vorticity(self, eps=0.05, iisph=False):
        """The force on the first step (gravity 0, so the acceleration is the force), at (0, 0) and after one divergence
        update (1, 0), each pass fed what its kernel read: omega on the velocities the forces saw and the step's densities,
        eta on the omega read back, the force on the omega and eta read back.  The force excludes (and counts) the particles
        whose eta bound reaches |eta| / 4, where N is ill-conditioned.  iisph: forces run on the velocities the step starts
        from (as in `artificial`), (0, 0) only."""
        ps, m, sc = self.ps, self.mutant, self.scene
        V0 = np.concatenate([f["velocities"] for f in sc["fluids"]]).astype(F)
        bvel = np.concatenate([b["velocities"] for b in sc["boundaries"]]).astype(F) if m == "vort_boundaries" else None
        for it, tag in (((0, 0), "_no_update"),) + ((((1, 0), "_after_update"),) if not iisph else ()):
            o, _ = S.run(self.make_world, sc, it, [(KIND, [eps])], extra=SCRATCH)
            om = omega(ps, V0 if iisph else o["V"], o["density"], C_PASS["vorticity_omega"], v_i_minus_v_j=m == "vort_v_i_minus_v_j",
                       rho_i=m == "vort_rho_i", any_fluid=m == "vort_other_fluids", bvel=bvel, bvol=o["bvol"])
            self.record("vorticity_omega" + tag, o["vorticity"], om, 0)
            et = eta(ps, o["density"], o["vorticity"], C_PASS["vorticity_eta"], plain_sum=m == "vort_eta_plain_sum")
            self.record("vorticity_eta" + tag, o["vorticity_eta"], et, 0)
            f = force(o["vorticity"], o["vorticity_eta"], eps, omega_x_n=m == "vort_omega_x_n", unnormalised=m == "vort_unnormalised")
            self.record("vorticity_force" + tag, o["acceleration"], f, C_PASS["vorticity_force"], exclude=ill_conditioned(et), ambiguous=False)
