"""oracle/ref64.py, the per-pass float64 reference, and the staging that feeds each pass its own inputs (oracle/ref64_stages.py),
checked without a GPU: the new reference agrees with the dense float32 restatement, the CPU oracle meets every bound on every
stage and scene, plausible kernel bugs applied to the reference are caught, and every edge scene reaches its edge."""
import numpy as np
import pytest

from oracle import ref64
from oracle import ref64_stages as S
from oracle.numpy_ref import NumpyDFSPH
from oracle.oracle import OracleWorld

H = float(np.float32(np.float32(S.R) * np.float32(2.0) * np.float32(2.0)))
FORCE_SCENES = ("block", "pairs", "two_fluids")


def _oracle(kd=0, kg=0):
    return lambda **kw: OracleWorld(S.R, 2.0, kernel_density=kd, kernel_gradient=kg, **kw)


def _checks(name, kd=0, kg=0, mutant=None):
    c = S.Checks(_oracle(kd, kg), S.SCENES[name](), kw=kd, kg=kg, mutant=mutant)
    c.stages()
    return c


@pytest.mark.parametrize("kd,kg", [(0, 0), (1, 2), (3, 1)], ids=["cubic", "poly6+spiky", "viscosity+poly6"])
def test_ref64_agrees_with_the_dense_float32_restatement(kd, kg):
    sc = S.scene_tail(129)
    ps = S.passes_for(sc, kw=kd, kg=kg)
    nd = NumpyDFSPH(S.R, 2.0, kernel_density=kd, kernel_gradient=kg)
    f = sc["fluids"][0]
    nd.add_fluid(f["positions"], f["density0"], velocities=f["velocities"])
    nd.add_boundary(sc["boundaries"][0]["positions"])
    nd.contacts()
    nd.densities_alphas()
    nd.divergences()
    assert np.array_equal(nd.nff, ps.nf) and np.array_equal(nd.nfb, ps.nb)
    assert ref64.ratio(1.0 / nd.bvol.astype(np.float64), ps.boundary_volume_sum(), ref64.C_PASS["boundary_volume"]).max() <= 1
    assert ref64.ratio(nd.dens, ps.density(nd.bvol), ref64.C_PASS["density"]).max() <= 1
    div = ps.divergence(f["velocities"], nd.bvol)
    assert ref64.ratio(nd.div, div, ref64.C_PASS["divergence"]).max() <= 1
    assert (div.value > 0).sum() >= 10


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_the_cpu_oracle_meets_every_bound(name):
    c = _checks(name)
    if name in FORCE_SCENES:
        c.akinci(0.0)
        c.akinci(0.5)
        c.xsph(0.5, 0.0)
        c.xsph(0.5, 0.3)
        c.artificial(1.0, 0.0)
        c.artificial(1.0, 0.5, beta=0.3)
    assert not c.flagged(), c.worst
    assert c.worst["counts"] == 0
    if name == "two_fluids":   # the walls want their forces: every boundary-force check ran
        assert {"boundary_force_first_step", "boundary_force_pressure", "boundary_force_adhesion", "boundary_force_xsph"} <= set(c.worst)


@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_the_cpu_oracle_meets_every_bound_with_generic_kernels(kd, kg):
    c = _checks("two_fluids", kd, kg)
    c.akinci(0.0)
    c.akinci(0.5)
    c.xsph(0.5, 0.3)
    c.artificial(1.0, 0.5, beta=0.3)
    assert not c.flagged(), c.worst


# mutant -> (scene it is meant for, the passes that must flag it)
MUTANTS = {
    "drop_entries_32_35": ("block", {"density", "divergence_sweep", "update", "divergence_eval", "pressure_update"}),
    "swap_vy_vz_odd": ("block", {"divergence_sweep", "divergence_eval", "predicted"}),
    "gate_at_21": ("gate", {"divergence_sweep", "divergence_eval"}),
    "normals_rho_i": ("two_fluids", {"akinci_unfused"}),
    "boundary_mass_fluid0_rho0": ("two_fluids", {"density", "alpha", "divergence_sweep", "update", "pressure_update"}),
    "no_kappa_gate": ("block", {"pressure_update"}),
    "drop_last_boundary": ("block", {"density", "divergence_sweep", "update", "pressure_update"}),
    "bforce_no_inv_dt": ("two_fluids", {"boundary_force_pressure"}),
    "artificial_no_vr_gate": ("block", {"artificial_no_update", "artificial_after_update"}),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_plausible_kernel_bugs_are_caught(mutant):
    scene, must = MUTANTS[mutant]
    c = _checks(scene, mutant=mutant)
    if mutant == "normals_rho_i":
        c.akinci(0.0)
    if mutant == "artificial_no_vr_gate":
        c.artificial(1.0, 0.5)
    flagged = set(c.flagged())
    assert must <= flagged, (flagged, c.worst)


def test_the_list_layout_scene_reaches_its_counts():
    for name in ("block", "far"):
        ps = S.passes_for(S.SCENES[name]())
        nf, nb = set(ps.nf.tolist()), set(ps.nb.tolist())
        assert {31, 32, 33, 35, 36, 37} <= nf, sorted(nf)
        assert {7, 8, 9} <= nb, sorted(nb)
        assert {n % 4 for n in nf} == {0, 1, 2, 3}
        assert max(nf) > 64                                   # beyond the initial list capacity: the lists regrow


def test_the_far_scene_has_negative_cells_and_coarse_coordinates():
    sc = S.scene_far()
    p = sc["fluids"][0]["positions"]
    assert (np.floor(p / H) < 0).any()
    assert np.spacing(np.abs(p).max()) >= 2.0 ** -14


def test_the_gate_scene_reaches_the_gate():
    sc = S.scene_gate()
    ps = S.passes_for(sc)
    v = sc["fluids"][0]["velocities"]
    bvol = 1.0 / ps.boundary_volume_sum().value
    ungated = ps.divergence(v, bvol, gate=False).value
    n = ps.nf + ps.nb
    for k in (19, 20, 21):
        assert ((n == k) & (ungated > 0)).sum() >= 5, k


def test_the_pair_scene_reaches_every_pair_edge():
    sc = S.scene_pairs()
    ps = S.passes_for(sc)
    ff, fb = ps.ff, ps.fb
    other = ff.i != ff.j
    eps2 = ref64.EPS32 ** 2
    t = ref64.grad_threshold(0, H)
    assert (other & (ff.d2 == 0)).sum() >= 2                   # coincident
    assert (other & (ff.d2 > 0) & (ff.d2 <= eps2)).sum() >= 1
    assert (other & (ff.d2 > eps2) & (ff.d2 <= t)).sum() >= 2  # Akinci cohesion acts, the gradient does not
    assert ((fb.d2 > eps2) & (fb.d2 <= t)).sum() >= 2
    P = ps.P
    h2 = np.float32(np.float32(H) * np.float32(H))
    d32 = ref64.f32_d2(P[ff.i], P[ff.j])
    assert (d32 == h2).sum() >= 2                              # exactly at the edge, both directions
    near = np.nonzero(np.abs(d32.astype(np.float64) - float(h2)) <= 2 ** -21 * float(h2))[0]
    fd = ref64.fma_d2(P[ff.i[near]], P[ff.j[near]])
    assert ((d32[near] <= h2) & (fd > h2)).sum() >= 2          # the fused d^2 lies on the other side
    assert not ps.ambiguous().any()


@pytest.mark.parametrize("n", S.TAILS)
def test_the_tail_scenes_have_their_sizes(n):
    ps = S.passes_for(S.scene_tail(n))
    assert ps.N == n
    if n == 1:
        assert ps.nf[0] == 1 and ps.nb[0] == 0                # self-only: gated, alpha = 0
