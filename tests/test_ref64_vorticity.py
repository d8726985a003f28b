"""Vorticity confinement's float64 reference (oracle/ref64_vorticity.py): its closed forms on a cubic lattice, the
CPU twin (ref64_vorticity.OracleVorticityWorld) against its bounds on every per-pass scene, and plausible kernel bugs applied to
the reference, each caught by the pass it corrupts."""
import numpy as np
import pytest

from oracle import ref64
from oracle import ref64_stages as S
from oracle import ref64_vorticity as V

F = np.float32
KERNELS = [(0, 0), (1, 2)]
KERNEL_IDS = ["cubic", "poly6+spiky"]


def _oracle(kd=0, kg=0, solver=0):
    return lambda **kw: V.OracleVorticityWorld(S.R, 2.0, solver=solver, kernel_density=kd, kernel_gradient=kg, **kw)


def _lattice(n=9, spacing=2 * S.R):
    """A full cubic lattice of n^3 particles centred on the origin, and the index of its centre."""
    a = (np.arange(n) - n // 2) * spacing
    P = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3).astype(F)
    return P, int(np.argmin((P.astype(np.float64) ** 2).sum(1)))


def _passes(P, kg):
    h = S.kernel_h(F(S.R), 2.0)
    N = len(P)
    m = np.full(N, F(1.0), F)
    return ref64.Passes(h, P, np.zeros(N, int), np.full(N, F(1000.0), F), m, np.zeros((0, 3), F), np.zeros(0, int), kg=kg)


def _interior(P, ps):
    """Particles whose whole kernel support lies inside the lattice."""
    x = np.abs(P.astype(np.float64)).max(1)
    return x + ps.h <= np.abs(P.astype(np.float64)).max() + 1e-9


def _kappa(ps, i, dens):
    """kappa = 1/3 sum_j V_j |grad W_ij| r_ij of particle i, in float64."""
    sel = ps.ff.i == i
    pr = ps.ff.subset(sel)
    g, _, _ = ps._g(pr)
    vol = ps.mass[pr.j] / dens[pr.j]
    return float((vol * np.abs(g) * pr.r * pr.r).sum() / 3.0)


def test_uniform_translation_has_no_vorticity():
    P, _ = _lattice(7)
    ps = _passes(P, 0)
    dens = np.full(len(P), 1000.0)
    om = V.omega(ps, np.tile(F([0.3, -1.2, 0.7]), (len(P), 1)), dens, 0)
    assert (om.value == 0).all()
    eta = V.eta(ps, dens, om.value, 0)
    assert (eta.value == 0).all()


@pytest.mark.parametrize("kd,kg", KERNELS, ids=KERNEL_IDS)
def test_rigid_rotation_gives_twice_kappa_omega(kd, kg):
    P, c = _lattice()
    ps = _passes(P, kg)
    dens = np.full(len(P), 1000.0)
    Om = np.array([0.4, -1.1, 0.7])
    vel = np.cross(Om, P.astype(np.float64))
    om = V.omega(ps, vel, dens, 0)   # float32 velocities, float64 sums: the lattice's symmetry holds to rounding
    kappa = _kappa(ps, c, dens)
    assert 0.5 < kappa < 2.0
    inside = _interior(P, ps)
    assert inside.sum() >= 27
    for i in np.flatnonzero(inside):
        np.testing.assert_allclose(om.value[i], 2 * _kappa(ps, i, dens) * Om, rtol=1e-6, atol=1e-6 * np.abs(Om).max())


@pytest.mark.parametrize("kd,kg", KERNELS, ids=KERNEL_IDS)
def test_linear_shear_gives_minus_gamma_kappa_z(kd, kg):
    P, c = _lattice()
    ps = _passes(P, kg)
    dens = np.full(len(P), 1000.0)
    gamma = 2.5
    vel = np.zeros((len(P), 3))
    vel[:, 0] = gamma * P[:, 1].astype(np.float64)
    om = V.omega(ps, vel, dens, 0)
    kappa = _kappa(ps, c, dens)
    np.testing.assert_allclose(om.value[c], [0.0, 0.0, -gamma * kappa], rtol=1e-6, atol=1e-9 * gamma * kappa)


def test_uniform_vorticity_magnitude_gives_no_eta():
    P, _ = _lattice(7)
    ps = _passes(P, 0)
    rng = np.random.default_rng(3)
    om = np.array([0.3, -1.7, 0.9]) * rng.choice([-1.0, 1.0], (len(P), 3))   # sign flips: |omega| the same bits everywhere
    eta = V.eta(ps, np.full(len(P), 1000.0), om, 0)
    assert (eta.value == 0).all()


@pytest.mark.parametrize("name", sorted(S.SCENES))
@pytest.mark.parametrize("kd,kg", KERNELS, ids=KERNEL_IDS)
def test_the_cpu_twin_meets_every_vorticity_bound(name, kd, kg):
    c = V.Checks(_oracle(kd, kg), S.SCENES[name](), kw=kd, kg=kg)
    c.vorticity(0.05)
    assert not c.flagged(), c.worst
    assert {"vorticity_omega_no_update", "vorticity_eta_no_update", "vorticity_force_no_update", "vorticity_omega_after_update",
            "vorticity_eta_after_update", "vorticity_force_after_update"} <= set(c.worst)


@pytest.mark.parametrize("name", ["block", "two_fluids", "volumes", "tail33"])
def test_the_cpu_twin_meets_every_vorticity_bound_under_iisph(name):
    c = V.Checks(_oracle(solver=1), S.SCENES[name]())
    c.vorticity(0.05, iisph=True)
    assert not c.flagged(), c.worst
    assert {"vorticity_omega_no_update", "vorticity_eta_no_update", "vorticity_force_no_update"} <= set(c.worst)


# mutant -> (scene, the passes that must flag it)
VORTICITY_MUTANTS = {
    "vort_v_i_minus_v_j": ("block", {"vorticity_omega_no_update", "vorticity_omega_after_update"}),
    "vort_rho_i": ("block", {"vorticity_omega_no_update", "vorticity_omega_after_update"}),
    "vort_other_fluids": ("two_fluids", {"vorticity_omega_no_update", "vorticity_omega_after_update"}),
    "vort_boundaries": ("block", {"vorticity_omega_no_update", "vorticity_omega_after_update"}),
    "vort_eta_plain_sum": ("block", {"vorticity_eta_no_update", "vorticity_eta_after_update"}),
    "vort_omega_x_n": ("block", {"vorticity_force_no_update", "vorticity_force_after_update"}),
    "vort_unnormalised": ("block", {"vorticity_force_no_update", "vorticity_force_after_update"}),
}


@pytest.mark.parametrize("mutant", sorted(VORTICITY_MUTANTS))
def test_plausible_vorticity_kernel_bugs_are_caught(mutant):
    """Each bound is smaller than the change the mutant makes, at the pass the mutant corrupts."""
    scene, must = VORTICITY_MUTANTS[mutant]
    c = V.Checks(_oracle(), S.SCENES[scene](), mutant=mutant)
    c.vorticity(0.05)
    assert must <= set(c.flagged()), c.worst


def test_the_block_scene_exercises_the_boundary_mutant():
    """The boundary mutant needs fluid-boundary contacts with moving boundaries."""
    sc = S.scene_block()
    ps = S.passes_for(sc)
    assert len(ps.fb.i) > 0
    assert np.abs(sc["boundaries"][0]["velocities"]).max() > 0


def test_the_selectors_are_refused_before_a_solve_and_after_an_append():
    from salva_b200 import scenes
    sc = S.scene_tail(33)
    w = _oracle()()
    fh, _ = S.populate(w, sc, [scenes.vorticity_confinement(0.05)])
    for sel in ("vorticity", "vorticity_eta"):
        with pytest.raises(AssertionError):
            w.debug(fh[0], sel)
    w.step(S.DT, S.ZERO_G)
    for sel in ("vorticity", "vorticity_eta"):
        assert w.debug(fh[0], sel).shape == (33, 3)
    w.append_particles(fh[0], np.array([[0.9, 0.9, 0.9]], F))
    for sel in ("vorticity", "vorticity_eta"):
        with pytest.raises(AssertionError):
            w.debug(fh[0], sel)


@pytest.mark.parametrize("eps", [0.0, -1.0, float("nan"), float("inf"), float("-inf")])
def test_the_cpu_twin_refuses_a_bad_eps(eps):
    from salva_b200 import scenes
    w = _oracle()()
    h = w.add_fluid(S.scene_tail(31)["fluids"][0]["positions"])
    with pytest.raises(AssertionError):
        w.push_force(h, *scenes.vorticity_confinement(eps))
