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


@pytest.mark.parametrize("kd,kg", [(0, 0), (1, 2), (3, 1)], ids=["cubic", "poly6+spiky", "viscosity+poly6"])
def test_iisph_passes_agree_with_the_dense_float32_restatement(kd, kg):
    """dii, aii, dij_pjl (fed p_1), p_2 and the velocity of numpy_ref.py's step_iisph, two pressure iterations, against the
    IISPH passes fed the dense restatement's own float32 values."""
    sc = S.scene_tail(129)
    ps = S.passes_for(sc, kw=kd, kg=kg)
    f = sc["fluids"][0]
    nds = []
    for k in (1, 2):
        nd = NumpyDFSPH(S.R, 2.0, kernel_density=kd, kernel_gradient=kg)
        nd.add_fluid(f["positions"], f["density0"], velocities=f["velocities"])
        nd.add_boundary(sc["boundaries"][0]["positions"], velocities=sc["boundaries"][0]["velocities"])
        nd.force_press = k
        nd.step_iisph(S.DT, S.ZERO_G)
        nds.append(nd)
    n1, n2 = nds
    C = ref64.C_PASS
    assert ref64.ratio(n2.dii, ps.iisph_dii(n2.dens, n2.bvol, S.DT), C["iisph_dii"]).max() <= 1
    assert ref64.ratio(n2.aii, ps.iisph_aii(n2.dens, n2.dii, n2.bvol, S.DT), C["iisph_aii"]).max() <= 1
    assert ref64.ratio(n2.dijpj, ps.iisph_dij_pjl(n2.dens, n1.press, S.DT), C["iisph_dij_pjl"]).max() <= 1
    ref, raw = ps.iisph_next_pressure(n2.dens, n2.pred, n1.press, n2.aii, n2.dii, n2.dijpj, n2.bvol, S.DT, 0.5)
    b = ref.bound(C["iisph_pressure"])
    clear = np.abs(np.nan_to_num(raw)) > b
    assert ref64.ratio(n2.press, ref, C["iisph_pressure"])[clear].max() <= 1
    assert (raw[clear] > 0).sum() >= 50 and (raw[clear] < 0).sum() >= 1     # both sides of the clamp
    v = ps.iisph_velocity(n2.dens, n2.press, f["velocities"], n2.bvol, S.DT)
    assert ref64.ratio(n2.V, v, C["iisph_velocity"]).max() <= 1
    assert (np.abs(v.value - f["velocities"]) > 100 * v.bound(C["iisph_velocity"])).any()


def _iisph(kd=0, kg=0):
    return lambda **kw: OracleWorld(S.R, 2.0, solver=1, kernel_density=kd, kernel_gradient=kg, **kw)


def _iisph_checks(name, kd=0, kg=0, mutant=None):
    c = S.Checks(_iisph(kd, kg), S.SCENES[name](), kw=kd, kg=kg, mutant=mutant)
    c.iisph_stages(alpha=False)   # the oracle's IISPH, like the reference's, computes no alpha
    return c


IISPH_PASSES = {"counts", "density", "predicted", "dii", "aii", "pressure_0", "pressure_1", "velocity", "dij_pjl", "pressure_2",
                "density_error", "dij_pjl_warm", "pressure_warm"}


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_the_cpu_oracle_meets_every_iisph_bound(name):
    c = _iisph_checks(name)
    assert not c.flagged(), c.worst
    assert IISPH_PASSES <= set(c.worst)
    assert c.worst["counts"] == 0
    if name == "two_fluids":
        assert "boundary_force_iisph" in c.worst
    if name == "block":   # the warm start is checked after most particles moved, many of them across cells
        assert c.moved_cells >= 300, c.moved_cells


@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_the_cpu_oracle_meets_every_iisph_bound_with_generic_kernels(kd, kg):
    c = _iisph_checks("two_fluids", kd, kg)
    assert not c.flagged(), c.worst


def test_the_iisph_pressure_clamp_is_reached_on_both_sides():
    """Particles whose unclamped pressure lies clear of 0 on each side, counted outside the excluded band."""
    c = _iisph_checks("block")
    for stage in ("pressure_1", "pressure_2", "pressure_warm"):
        below, above = c.clamp[stage]
        assert below >= 1 and above >= 1000, (stage, c.clamp)
    assert _iisph_checks("gate").clamp["pressure_2"][0] >= 1000   # almost every particle clamped


IISPH_MUTANTS = {
    "dji_mass_j": ("volumes", {"aii", "pressure_2"}),
    "s_without_dii_p": ("block", {"pressure_2"}),
    "dij_prho_i": ("block", {"dij_pjl"}),
    "next_p_no_boundary": ("block", {"pressure_2"}),
    "no_relaxation": ("block", {"pressure_2"}),
    "boundary_mass_fluid0_rho0": ("two_fluids", {"dii", "aii", "pressure_1", "velocity"}),
    "velocity_prho_i_twice": ("block", {"velocity"}),
    "no_warm_start": ("block", {"dij_pjl_warm", "pressure_warm"}),
    "error_counts_clamped": ("block", {"density_error"}),
    "iisph_bforce_no_mass": ("two_fluids", {"boundary_force_iisph"}),
}


@pytest.mark.parametrize("mutant", sorted(IISPH_MUTANTS))
def test_plausible_iisph_kernel_bugs_are_caught(mutant):
    scene, must = IISPH_MUTANTS[mutant]
    flagged = set(_iisph_checks(scene, mutant=mutant).flagged())
    assert must <= flagged, flagged


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


TENSION_SCENES = ("block", "pairs", "two_fluids", "volumes", "tail1", "tail33")


def _tension(c):
    c.wcsph(0.5)
    for cf, cb in ((0.5, 0.0), (0.0, 0.3), (0.5, 0.3)):
        c.he2014(cf, cb)
    return c


@pytest.mark.parametrize("name", TENSION_SCENES)
def test_the_cpu_oracle_meets_every_surface_tension_bound(name):
    c = _tension(S.Checks(_oracle(), S.SCENES[name]()))
    assert not c.flagged(), c.worst
    assert {"wcsph", "he2014_color", "he2014_gradc", "he2014_force_fluid", "he2014_force_boundary", "he2014_force_both"} <= set(c.worst)
    if name == "two_fluids":   # the walls want their forces: He2014's reaction is checked
        assert "boundary_force_he2014" in c.worst


@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_the_cpu_oracle_meets_every_surface_tension_bound_with_generic_kernels(kd, kg):
    c = _tension(S.Checks(_oracle(kd, kg), S.SCENES["two_fluids"](), kw=kd, kg=kg))
    assert not c.flagged(), c.worst


def test_the_he2014_gradc_bound_is_not_vacuous():
    """gradc's bound is carried through the cancelling vector sum explicitly; it stays far below gradc where the colour
    gradient does not cancel (the free surface), so a relative error of a few percent there is caught."""
    from salva_b200 import scenes
    sc = S.scene_block()
    w = _oracle()()
    fh, _ = S.populate(w, sc, [scenes.he2014_surface_tension(0.5, 0.0)])
    w.force_iterations(0, 0)
    w.step(S.DT, S.ZERO_G)
    ps = S.passes_for(sc)
    ref = ps.he2014_gradc(w.debug(fh[0], "density"), w.debug(fh[0], "he2014_color"), ref64.C_PASS["he2014_gradc"])
    surface = ref.value > np.quantile(ref.value, 0.9)
    assert (ref.bound(0)[surface] < 1e-3 * ref.value[surface]).all()


# mutant -> (scene, the passes that must flag it)
TENSION_MUTANTS = {
    "wcsph_inverted_mass_ratio": ("volumes", {"wcsph"}),
    "he2014_colors_no_boundary": ("block", {"he2014_color"}),
    "he2014_gradc_by_cj": ("block", {"he2014_gradc"}),
    "he2014_gradc_i_twice": ("block", {"he2014_force_fluid", "he2014_force_both"}),
    "he2014_reaction_sign": ("two_fluids", {"boundary_force_he2014"}),
}


@pytest.mark.parametrize("mutant", sorted(TENSION_MUTANTS))
def test_plausible_surface_tension_kernel_bugs_are_caught(mutant):
    scene, must = TENSION_MUTANTS[mutant]
    flagged = set(_tension(S.Checks(_oracle(), S.SCENES[scene](), mutant=mutant)).flagged())
    assert must <= flagged, flagged


BECKER_SCENES = ("block", "two_fluids", "volumes")


def _becker(c):
    c.becker(nonlinear=True)
    c.becker(nonlinear=False)
    return c


@pytest.mark.parametrize("name", BECKER_SCENES)
def test_the_cpu_oracle_meets_every_becker_bound(name):
    c = _becker(S.Checks(_oracle(), S.SCENES[name]()))
    assert not c.flagged(), c.worst
    for stage in ("el_rest", "el_deformed", "el_warm", "el_recaptured"):
        for kind in ("nonlinear", "linear"):
            assert {"%s_%s_%s" % (stage, kind, p) for p in ("rotation", "orthonormal", "grad_tr", "stress", "force")} <= set(c.worst)
    # the deformation turned every checked particle by more than 20 degrees, some over many iterations; the float64 run
    # ends on the polar rotation; the current contacts differ from the rest contacts for many particles
    assert c.el_turn >= 20 and c.el_iterations >= 5, (c.el_turn, c.el_iterations)
    assert c.el_polar_gap <= 1e-6, c.el_polar_gap
    assert c.rest_differs >= 100, c.rest_differs
    assert "el_recaptured_volume" in c.worst


def test_the_cpu_oracle_meets_every_becker_bound_under_iisph():
    """Becker runs under IISPH in the C5 configuration."""
    c = _becker(S.Checks(_iisph(), S.SCENES["two_fluids"]()))
    assert not c.flagged(), c.worst
    assert max(v for k, v in c.excluded.items() if k.endswith("rotation")) <= 0.05 * c.ps.N, c.excluded   # per stage


def test_the_becker_rest_lists_exceed_the_initial_capacity():
    sc = S.scene_block()
    ps = S.passes_for(sc)
    bk = ref64.Becker(ps.h, ps.P, ps.fid, ps.mass, 2e5, 0.3, True)
    assert bk.n.max() > 64


BECKER_MUTANTS = {
    "el_volume_once": ("block", {"el_volume"}),
    "el_r_i_for_r_j": ("block", {"el_deformed_nonlinear_force", "el_deformed_linear_force"}),
    "el_g_i_for_g_j": ("block", {"el_deformed_nonlinear_force"}),
    "el_rest_lists_recaptured": ("two_fluids", {"el_deformed_nonlinear_rotation", "el_deformed_nonlinear_grad_tr",
                                                "el_deformed_nonlinear_force"}),
    "el_second_fluid_no_offset": ("two_fluids", {"el_deformed_nonlinear_rotation", "el_deformed_nonlinear_grad_tr"}),
    # the old rest volumes are about 1e-7 of the sum at water's density, below float32's resolution: a light fluid
    "el_recapture_no_old_volumes": ("light_two_fluids", {"el_recaptured_volume"}),
}


def _scene(name):
    return S.light(S.SCENES[name[6:]]()) if name.startswith("light_") else S.SCENES[name]()


@pytest.mark.parametrize("mutant", sorted(BECKER_MUTANTS))
def test_plausible_becker_kernel_bugs_are_caught(mutant):
    scene, must = BECKER_MUTANTS[mutant]
    flagged = set(_becker(S.Checks(_oracle(), _scene(scene), mutant=mutant)).flagged())
    assert must <= flagged, flagged


# DFSPHViscosity: on light fluids beta is non-zero everywhere; at water's density (block) and for a lone particle (tail1)
# the determinant gate sets it to 0
VISC_SCENES = ("light_block", "light_two_fluids", "light_volumes", "block", "tail1")


def _visc(c):
    c.viscosity(0.5)
    c.viscosity(0.5, wcsph=2.0)
    return c


@pytest.mark.parametrize("name", VISC_SCENES)
def test_the_cpu_oracle_meets_every_viscosity_bound(name):
    c = _visc(S.Checks(_oracle(), _scene(name)))
    assert not c.flagged(), c.worst
    assert {"visc_beta", "visc_beta_gate", "visc_target", "visc_accel_1", "visc_accel_2", "visc_target_after_wcsph",
            "visc_accel_2_after_wcsph"} <= set(c.worst)
    if name.startswith("light_"):
        assert c.visc_zero == 0 and sum(c.excluded.values()) <= 4, (c.visc_zero, c.excluded)
    else:   # most particles on the beta = 0 path, the gate checked for each
        assert c.visc_zero >= c.ps.N, c.visc_zero


VISC_MUTANTS = {
    "visc_precondition_columns": ("light_block", {"visc_beta"}),
    "visc_target_no_scale": ("light_block", {"visc_target"}),
    "visc_vv_no_adt": ("light_block", {"visc_target_after_wcsph", "visc_accel_1_after_wcsph", "visc_accel_2"}),
    "visc_u_j_beta_i": ("light_block", {"visc_accel_1", "visc_accel_2"}),
}


@pytest.mark.parametrize("mutant", sorted(VISC_MUTANTS))
def test_plausible_viscosity_kernel_bugs_are_caught(mutant):
    scene, must = VISC_MUTANTS[mutant]
    flagged = set(_visc(S.Checks(_oracle(), _scene(scene), mutant=mutant)).flagged())
    assert must <= flagged, flagged


def test_the_plugin_scratch_is_refused_without_its_force():
    """The CPU oracle's selectors 12-19 refuse a fluid without the force, or before it has been solved; with it they have
    one row of the selector's width per particle."""
    from salva_b200 import scenes
    sc = S.scene_tail(33)
    kinds = {"he2014": scenes.he2014_surface_tension(0.5, 0.3), "visc": scenes.dfsph_viscosity(0.1),
             "el": scenes.becker2009_elasticity(1e5, 0.3)}
    sel = {"he2014_color": ("he2014", ()), "he2014_gradc": ("he2014", ()), "visc_beta": ("visc", (36,)),
           "visc_target": ("visc", (6,)), "el_volume0": ("el", ()), "el_rotation": ("el", (9,)), "el_grad_tr": ("el", (9,)),
           "el_stress": ("el", (6,))}
    for kind, force in kinds.items():
        for stage in ("pushed", "stepped", "written"):
            w = _oracle()()
            (fh,), _ = S.populate(w, sc, [force])
            if stage != "pushed":
                w.step(S.DT, S.ZERO_G)
            if stage == "written":   # same particles, new positions: the last solve's scratch stays readable
                w.write_fluid(fh, positions=w.read_fluid(fh)[0])
            for what, (k, shape) in sel.items():
                if k == kind and stage in ("stepped", "written"):
                    assert w.debug(fh, what).shape == (33,) + shape
                else:
                    with pytest.raises(AssertionError):
                        w.debug(fh, what)


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
