"""The rows mode of oracle/ref64.py (contacts of a sample of particles only, which is what lets the per-pass reference reach
the benchmark's sizes) and the structural bound of the loop-error reductions, checked without a GPU:
  - on every edge scene, every pass evaluated in rows mode is bit-identical at the rows (value, A, K and n) to the full
    evaluation: the same contacts in the same order give the same float64 terms summed in the same order;
  - the plausible kernel bugs of tests/test_ref64.py, applied to the reference in rows mode, are still flagged by the same
    passes;
  - on 10 077 696 terms in 78 732 blocks (C3's evaluation), the structural bound holds for a float32 emulation of the
    kernels' reduction tree, and flags the loss of every partial past block 65 535, which the any-order bound lets pass."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import ref64
from oracle import ref64_stages as S
from test_ref64 import IISPH_MUTANTS, MUTANTS, _iisph, _oracle

F = np.float32


def _rows(sc, frac, seed, boundary=12):
    """A seeded sample of a scene's particles: a fraction of them at random, plus every fluid particle near a few random
    boundary particles (so that some boundary particles have all their fluid contacts among the rows)."""
    ps = S.passes_for(sc)
    rng = np.random.default_rng(seed)
    pick = [np.nonzero(rng.random(ps.N) < frac)[0]]
    if len(ps.BP):
        b = rng.choice(len(ps.BP), size=min(boundary, len(ps.BP)), replace=False)
        near = cKDTree(ps.P.astype(np.float64)).query_ball_point(ps.BP[b].astype(np.float64), ps.h * (1 + 1e-5))
        pick += [np.asarray(x, np.int64) for x in near]
    rows = np.unique(np.concatenate(pick))
    return rows if len(rows) else np.array([0])


def _same(name, a, b, at):
    for f in ("value", "A", "K", "n"):
        x, y = getattr(a, f), getattr(b, f)
        assert np.array_equal(x[at], y[at]), (name, f)


def _inputs(ps, sc, seed):
    """Float32 inputs of the passes, as a kernel would read them: densities around rest, velocities, kappas, pressures,
    dii and dij_pjl, and boundary volumes and velocities."""
    rng = np.random.default_rng(seed)
    N, nb = ps.N, len(ps.BP)
    f = lambda a: np.asarray(a, F)  # noqa: E731
    return dict(dens=f(ps.rho0 * rng.uniform(0.9, 1.2, N)), V=f(np.concatenate([x["velocities"] for x in sc["fluids"]])),
                kappa=f(rng.uniform(-5, 20, N)), press=f(rng.uniform(0, 300, N)), dii=f(rng.normal(0, 1e-6, (N, 3))),
                dij=f(rng.normal(0, 1e-4, (N, 3))), aii=f(rng.uniform(-2e-6, -1e-7, N)),
                bvol=f(1.0 / ps.boundary_volume_sum().value) if nb else np.zeros(0, F), bvel=f(rng.normal(0, 0.1, (nb, 3))))


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_every_pass_in_rows_mode_is_bit_identical_at_the_rows(name):
    sc = S.SCENES[name]()
    rows = _rows(sc, 0.3, 5)
    full, part = S.passes_for(sc), S.passes_for(sc, rows=rows)
    x = _inputs(full, sc, 11)
    dens, V, bvol, bvel, dt = x["dens"], x["V"], x["bvol"], x["bvel"], S.DT
    inv_dt = F(1.0) / F(dt)
    assert np.array_equal(full.nf[rows], part.nf[rows]) and np.array_equal(full.nb[rows], part.nb[rows])
    assert np.array_equal(full.ambiguous()[rows], part.ambiguous()[rows])
    calls = {
        "density": lambda p: p.density(bvol),
        "alpha": lambda p: p.den(bvol),
        "divergence": lambda p: p.divergence(V, bvol),
        "predicted": lambda p: p.divergence(V, bvol, predicted=True, bvel=bvel, dens=dens, dt=dt),
        "update": lambda p: p.update(x["kappa"], bvol, V),
        "pressure_update": lambda p: p.update(x["kappa"], bvol, V, pressure=True, inv_dt=inv_dt),
        "iisph_dii": lambda p: p.iisph_dii(dens, bvol, dt),
        "iisph_aii": lambda p: p.iisph_aii(dens, x["dii"], bvol, dt),
        "iisph_dij_pjl": lambda p: p.iisph_dij_pjl(dens, x["press"], dt),
        "iisph_pressure": lambda p: p.iisph_next_pressure(dens, dens, x["press"], x["aii"], x["dii"], x["dij"], bvol, dt, 0.5)[0],
        "iisph_velocity": lambda p: p.iisph_velocity(dens, x["press"], V, bvol, dt),
        "akinci": lambda p: p.akinci(dens, 1.0, 0.5, bvol),
        "xsph": lambda p: p.xsph(V, dens, 0.5, 0.3, inv_dt, bvel, bvol),
        "artificial": lambda p: p.artificial(V, dens, 1.0, 0.5, 1.0, 0.3, 10.0, bvel, bvol)[0],
    }
    for what, call in calls.items():
        _same(what, call(full), call(part), rows)
    _, amb_f = full.artificial(V, dens, 1.0, 0.5, 1.0, 0.3, 10.0, bvel, bvol)
    _, amb_p = part.artificial(V, dens, 1.0, 0.5, 1.0, 0.3, 10.0, bvel, bvol)
    assert np.array_equal(amb_f[rows], amb_p[rows])
    # sums onto boundary particles: whole at brows
    if len(full.BP):
        _same("boundary_volume", full.boundary_volume_sum(), part.boundary_volume_sum(), slice(None))
        _same("pressure_boundary_force", full.pressure_boundary_force(x["kappa"], bvol, inv_dt),
              part.pressure_boundary_force(x["kappa"], bvol, inv_dt), part.brows)
    # Becker2009 at the capture: rest volumes, A_pq, grad_tr, stress and force on the rest contacts
    Q = full.P
    R = np.tile(np.eye(3), (full.N, 1, 1)) + np.random.default_rng(3).normal(0, 1e-3, (full.N, 3, 3))
    vol0 = (full.mass / full.rho0).astype(F)
    G = np.random.default_rng(4).normal(0, 1e-3, (full.N, 3, 3)).astype(F)
    Sg = np.random.default_rng(5).normal(0, 10.0, (full.N, 6)).astype(F)
    bf, bp = (ref64.Becker(full.h, Q, full.fid, full.mass, 1e5, 0.3, True, rows=r) for r in (None, rows))
    _same("el_volume", bf.volume_sum(), bp.volume_sum(), rows)
    for a, b in zip(bf.apq(Q, 18), bp.apq(Q, 18)):
        assert np.array_equal(a[rows], b[rows])
    _same("el_grad_tr", bf.grad_tr(Q, R, vol0), bp.grad_tr(Q, R, vol0), rows)
    _same("el_force", bf.force(Sg, G, R, vol0), bp.force(Sg, G, R, vol0), rows)


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_plausible_kernel_bugs_are_caught_in_rows_mode(mutant):
    scene, must = MUTANTS[mutant]
    sc = S.SCENES[scene]()
    c = S.Checks(_oracle(), sc, mutant=mutant, rows=_rows(sc, 0.5, 7, boundary=40))
    c.stages()
    if mutant == "normals_rho_i":
        c.akinci(0.0)
    if mutant == "artificial_no_vr_gate":
        c.artificial(1.0, 0.5)
    flagged = set(c.flagged())
    assert must <= flagged, (flagged, c.worst)


@pytest.mark.parametrize("mutant", sorted(m for m in IISPH_MUTANTS if m != "error_counts_clamped"))
def test_plausible_iisph_kernel_bugs_are_caught_in_rows_mode(mutant):
    """error_counts_clamped shows only in the density error, a sum over every particle that rows mode does not check."""
    scene, must = IISPH_MUTANTS[mutant]
    sc = S.SCENES[scene]()
    c = S.Checks(_iisph(), sc, mutant=mutant, rows=_rows(sc, 0.5, 7, boundary=40))
    c.iisph_stages(alpha=False)
    flagged = set(c.flagged())
    assert must <= flagged, (flagged, c.worst)


def test_the_oracle_meets_every_bound_in_rows_mode():
    """The CPU oracle against rows mode on the two-fluid scene: every pass, the forces and the IISPH passes pass."""
    sc = S.scene_two_fluids()
    rows = _rows(sc, 0.4, 9, boundary=40)
    c = S.Checks(_oracle(), sc, rows=rows)
    c.stages()
    c.akinci(0.0)
    c.akinci(0.5)
    c.xsph(0.5, 0.3)
    c.artificial(1.0, 0.5, beta=0.3)
    assert not c.flagged(), c.worst
    assert {"counts", "density", "alpha", "update", "pressure_update", "akinci_unfused", "boundary_force_pressure"} <= set(c.worst)
    ci = S.Checks(_iisph(), sc, rows=rows)
    ci.iisph_stages(alpha=False)
    assert not ci.flagged(), ci.worst


def test_the_scene_radius_and_dt_are_the_scene_s_own():
    sc = dict(S.scene_tail(33), particle_radius=0.025, dt=0.001)
    ps = S.passes_for(sc)
    assert ps.h == float(F(F(0.025) * F(2.0) * F(2.0)))
    assert ps.mass[0] == float(F(F(0.025) ** 3 * F(8.0 * 0.8)) * F(1000.0))
    c = S.Checks(_oracle(), sc)
    assert (c.r, c.dt) == (0.025, 0.001)
    assert S.passes_for(S.scene_tail(33)).h == float(F(F(S.R) * F(2.0) * F(2.0)))


# ---- the structural loop-error bound at C3's size -------------------------------------------------------------------------
N_C3 = 10_077_696


@pytest.fixture(scope="module")
def c3_terms():
    """10 077 696 float32 error terms like a divergence evaluation's: max(d, 0) / rho0, 40 % of them gated to 0."""
    rng = np.random.default_rng(2024)
    e = rng.exponential(1e-3, N_C3).astype(F)
    e[rng.random(N_C3) < 0.4] = 0
    return e


def test_the_c3_reduction_has_its_derived_depth():
    assert -(-N_C3 // S.PASS_T) == 78_732 > 65_536
    assert ref64.structural_depth(N_C3, S.PASS_T, S.PASS_T) == 7 + 615 + 7
    assert ref64.structural_depth(N_C3, S.NBR_T, S.REDUCE_T) == 7 + 307 + 8
    assert ref64.structural_depth(100, 128, 128) == 14        # one block: two trees, no strided sums


@pytest.mark.parametrize("second", [S.PASS_T, S.REDUCE_T], ids=["last_block", "reduce_partials"])
def test_the_structural_bound_holds_for_the_kernels_tree(c3_terms, second):
    e = c3_terms
    exact = e.astype(np.float64).sum()
    got, part = ref64.emulate_reduction(e, S.PASS_T, second)
    assert len(part) == 78_732
    D = ref64.structural_depth(len(e), S.PASS_T, second)
    bound = D * ref64.U / (1 - D * ref64.U) * np.abs(e.astype(np.float64)).sum()
    err = abs(float(got) - exact)
    assert err <= bound, (err, bound)
    # losing every partial of block >= 65 536 is far outside it; the any-order bound (n + 4) u sum |e| lets it pass
    lost = part[65_536:].astype(np.float64).sum()
    assert lost > 1000 * bound
    assert lost < (len(e) + 4) * ref64.U * exact
    # one lost block of 128 terms lies below the structural bound at this size (the small scenes' mutant covers it)
    assert part[-1] < bound


def test_the_structural_bound_is_not_the_any_order_one(c3_terms):
    """A plain left-to-right float32 sum of the same terms (depth n) lies outside the structural bound: the depth it
    counts is the kernels', not any order's."""
    e = c3_terms[:2_000_000]
    exact = e.astype(np.float64).sum()
    seq = np.cumsum(e, dtype=F)[-1]
    D = ref64.structural_depth(len(e), S.PASS_T, S.PASS_T)
    assert abs(float(seq) - exact) > D * ref64.U * exact


def test_the_oracle_meets_the_c5_stages_in_rows_mode():
    """What the full-size C5 check runs, on the two-fluid scene under IISPH in rows mode: the IISPH passes, artificial
    viscosity on the velocities the step starts from (IISPH runs its forces before the pressure solve), and Becker2009 at
    the capture."""
    sc = S.scene_two_fluids()
    c = S.Checks(_iisph(), sc, rows=_rows(sc, 0.4, 13, boundary=40))
    c.iisph_stages(alpha=False)
    c.artificial(1.0, 0.0, iisph=True)
    c.artificial(1.0, 0.5, beta=0.3, iisph=True)
    c.becker_capture(1.0e5, 0.3, True)
    c.becker_capture(1.0e5, 0.3, False)
    assert not c.flagged(), c.worst
    assert {"artificial_no_update", "el_volume", "el_capture_nonlinear_force", "el_capture_linear_stress"} <= set(c.worst)
