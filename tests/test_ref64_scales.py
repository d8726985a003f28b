"""The float64 per-pass checks (oracle/ref64_stages.py) away from particle radius 0.05 and smoothing factor 2, checked without a
GPU: the CPU oracle meets every bound on every scale scene, the kernel bugs those scenes are built for, applied to the
reference, are caught by them, and each scene reaches the regime it is built for."""
import numpy as np
import pytest

from oracle import ref64
from oracle import ref64_stages as S
from oracle.oracle import OracleWorld

F = np.float32
NAMES = sorted(S.SCALE_SCENES)


def _oracle(sc, kd=0, kg=0, solver=0):
    return lambda **kw: OracleWorld(S.radius(sc), S.smoothing(sc), solver=solver, kernel_density=kd, kernel_gradient=kg, **kw)


def _checks(name, kd=0, kg=0, mutant=None, solver=0, light=False):
    sc = S.SCALE_SCENES[name]()
    sc = S.light(sc) if light else sc
    return S.Checks(_oracle(sc, kd, kg, solver), sc, kw=kd, kg=kg, mutant=mutant)


@pytest.mark.parametrize("name", NAMES)
def test_the_cpu_oracle_meets_every_bound(name):
    c = _checks(name)
    c.stages()
    c.akinci(0.0)
    c.akinci(0.5)
    c.xsph(0.5, 0.3)
    c.artificial(1.0, 0.5, beta=0.3)
    c.wcsph(0.5)
    c.he2014(0.5, 0.3)
    c.loop_errors()
    assert not c.flagged(), c.worst
    assert c.worst["counts"] == 0


@pytest.mark.parametrize("name", NAMES)
def test_the_cpu_oracle_meets_every_iisph_viscosity_and_becker_bound(name):
    c = _checks(name, solver=1)
    c.iisph_stages(alpha=False)   # the oracle's IISPH computes no alpha
    assert not c.flagged(), c.worst
    v = _checks(name, light=True)
    v.viscosity(0.5)
    assert not v.flagged(), v.worst
    b = _checks(name)
    b.becker(nonlinear=True)
    assert not b.flagged(), b.worst


@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_the_cpu_oracle_meets_every_bound_with_generic_kernels_at_small_h(kd, kg):
    """poly6_n, spiky_n and visc_n carry up to h^-9: at h = 0.008 they are the largest normalisations any scene reaches."""
    c = _checks("small", kd, kg)
    c.stages()
    c.akinci(0.5)
    c.he2014(0.5, 0.3)
    assert not c.flagged(), c.worst


# mutant -> (scene it is meant for, the passes that must flag it)
MUTANTS = {
    "grad_threshold_h_only": ("small", {"dii", "aii"}),
    "drop_entries_256_259": ("sf3", {"density", "divergence_sweep", "update", "divergence_eval", "pressure_update"}),
    # a tie sits at q = 1, where every kernel and its gradient vanish: the counts (and the gate they feed) show it
    "ties_excluded": ("sf1_lattice", {"counts"}),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_plausible_kernel_bugs_are_caught(mutant):
    scene, must = MUTANTS[mutant]
    assert mutant in S.MUTANTS
    if mutant == "grad_threshold_h_only":   # the gradient alone, with no contact gate before it: IISPH's dii and aii
        c = _checks(scene, mutant=mutant, solver=1)
        c.iisph_stages(alpha=False)
    else:
        c = _checks(scene, mutant=mutant)
        c.stages()
    flagged = set(c.flagged())
    assert must <= flagged, (flagged, c.worst)


def test_the_scale_scenes_form_h_as_the_engine_does():
    for name, want in (("sf1_lattice", 0.125), ("sf3", 0.3), ("sf_odd", 0.137), ("small", 0.008)):
        sc = S.SCALE_SCENES[name]()
        r, sf = S.radius(sc), S.smoothing(sc)
        h = S.passes_for(sc).h
        assert h == float(F(F(F(r) * F(sf)) * F(2.0))) and abs(h - want) <= 1e-7, name
    assert S.smoothing(S.scene_block()) == 2.0 and S.passes_for(S.scene_block()).h == float(F(0.2))


def test_the_sf1_lattice_scene_ties_every_axis_pair_and_reaches_the_gate():
    sc = S.scene_sf1_lattice()
    ps = S.passes_for(sc)
    n_lat = sc["lattice"]
    P = ps.P
    assert (P[:n_lat] * 16).astype(np.float64).tolist() == np.round(P[:n_lat] * 16).tolist()   # odd multiples of 2^-4
    h2 = F(F(ps.h) * F(ps.h))
    assert float(h2) == 2.0 ** -6
    d32 = ref64.f32_d2(P[ps.ff.i], P[ps.ff.j])
    lat = (ps.ff.i < n_lat) & (ps.ff.j < n_lat)
    assert ((d32 == h2) & lat).sum() == S.lattice_ties(S.SF1_LATTICE)
    assert (ps.nf[:n_lat] == 7).sum() >= 100                           # self and six ties
    assert ((ref64.f32_d2(P[ps.fb.i], ps.BP[ps.fb.j]) == h2).sum()) >= 100   # the walls, at d^2 = h^2 too
    v = sc["fluids"][0]["velocities"]
    bvol = 1.0 / ps.boundary_volume_sum().value
    ungated = ps.divergence(v, bvol, gate=False).value
    n = ps.nf + ps.nb
    for k in (19, 20, 21):
        assert ((n == k) & (ungated > 0)).sum() >= 5, k
    assert not ps.ambiguous().any()


def test_the_sf3_scene_regrows_its_lists_past_256():
    ps = S.passes_for(S.scene_sf3())
    assert ps.nf.max() > 256 and (ps.nf > 259).sum() >= 100
    assert ps.nb.max() >= 32
    assert not ps.ambiguous().any()


def test_the_sf_odd_scene_splits_at_the_gate_on_irregular_cell_faces():
    sc = S.scene_sf_odd()
    ps = S.passes_for(sc)
    n = ps.nf + ps.nb
    assert (n < 20).sum() >= 100 and (n >= 20).sum() >= 100
    frac = np.mod(ps.P.astype(np.float64) / ps.h, 1.0)    # positions within their cells: no lattice alignment
    assert np.histogram(frac[:, 0], bins=8, range=(0, 1))[0].min() >= 50


def test_the_small_scene_reaches_the_eps_gate():
    sc = S.scene_small()
    ps = S.passes_for(sc)
    eps2, t_h = ref64.EPS32 ** 2, float(F((1e-5 * ps.h) ** 2))
    assert ps.grad_t == float(F(eps2)) and t_h < eps2               # the eps^2 branch of the gate
    ff, fb = ps.ff, ps.fb
    other = ff.i != ff.j
    band = other & (ff.d2 > t_h) & (ff.d2 <= eps2)
    assert (other & (ff.d2 == 0)).sum() >= 2                         # coincident
    assert (other & (ff.d2 > 0) & (ff.d2 <= t_h)).sum() >= 1
    assert band.sum() >= 4                                           # both directions of two pairs in the block
    assert ((fb.d2 > t_h) & (fb.d2 <= eps2)).sum() >= 2
    a, b = sc["isolated"]
    assert ps.nf[a] == ps.nf[b] == 2 and ps.nb[a] == ps.nb[b] == 0   # each other and themselves only
    assert band[ff.i == a].sum() == 1
    h2 = F(F(ps.h) * F(ps.h))
    d32 = ref64.f32_d2(ps.P[ff.i], ps.P[ff.j])
    assert (d32 == h2).sum() >= 2
    near = np.nonzero(np.abs(d32.astype(np.float64) - float(h2)) <= 2 ** -21 * float(h2))[0]
    fd = ref64.fma_d2(ps.P[ff.i[near]], ps.P[ff.j[near]])
    assert ((d32[near] <= h2) & (fd > h2)).sum() >= 2
    assert not ps.ambiguous().any()
    # with the h-only threshold the isolated pair has a gradient
    ps.grad_t = t_h
    g, _, _ = ps._g(ff)
    assert (g[(ff.i == a) & other] != 0).all()
