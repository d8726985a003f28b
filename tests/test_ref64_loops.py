"""The DFSPH loop errors, the loops' exits, the lagging dt and the state a step carries into the next (oracle/ref64.py,
oracle/ref64_stages.py: Checks.loop_errors, .loop_exits, .lagging_dt, .grid_growth), checked without a GPU: the CPU oracle
meets every bound on every scene, plausible kernel bugs applied to the reference are caught, and the scenes reach their
edges."""
import numpy as np
import pytest

from oracle import ref64_stages as S
from oracle.oracle import OracleWorld

DT = S.DT


def _oracle(**kw):
    return OracleWorld(S.R, 2.0, **kw)


def _checks(name, mutant=None):
    return S.Checks(_oracle, S.LOOP_SCENES[name](), mutant=mutant)


@pytest.mark.parametrize("name", sorted(S.LOOP_SCENES))
def test_the_cpu_oracle_meets_every_loop_error_bound(name):
    c = _checks(name)
    c.loop_errors()
    c.loop_errors((DT, 2 * DT))
    assert not c.flagged(), c.worst
    for e in ("divergence_error", "density_error"):
        assert {e, e + "_read", e + "_after_dt_change", e + "_read_after_dt_change"} <= set(c.worst)
    # every evaluation's error is nonzero, and on the first step every non-empty fluid adds nonzero terms to it, so that a
    # dropped per-fluid partial shows (gate and tail33 lie below rest density: their density errors may be 0)
    if name in ("block", "two_fluids", "sixteen"):
        assert min(min(v) for v in c.errors.values()) > 0, c.errors
        assert c.nonzero["divergence"] >= 1 and c.nonzero["density"] >= 1, c.nonzero


def test_the_sixteen_fluid_scene_meets_every_pass_bound():
    """All sixteen fluid slots, one of them emptied by a delete, under the DFSPH and the IISPH passes."""
    sc = S.scene_sixteen()
    assert len(sc["fluids"]) == 16 and len(sc["fluids"][S.SIXTEEN_EMPTIED]["positions"]) == 0
    n = [len(f["positions"]) for f in sc["fluids"] if len(f["positions"])]
    assert min(n) == 1 and max(n) >= 250
    c = S.Checks(_oracle, sc)
    c.stages()
    assert not c.flagged(), c.worst
    ci = S.Checks(lambda **kw: OracleWorld(S.R, 2.0, solver=1, **kw), sc)
    ci.iisph_stages(alpha=False)
    assert not ci.flagged(), ci.worst
    # the group cuts remove fluid pairs that are in range
    every = S.ref64.contacts(c.ps.P, c.ps.P, c.ps.h, lambda i, j: np.ones(len(i), bool), same=True)
    assert len(every.i) - len(c.ps.ff.i) >= 100


@pytest.mark.parametrize("name", ["block", "two_fluids", "sixteen"])
def test_the_cpu_oracle_meets_every_lagging_dt_bound(name):
    c = _checks(name)
    c.lagging_dt()
    assert not c.flagged(), c.worst
    assert {"carried_divergence", "lagging_update", "lagging_boundary_force_divergence", "lagging_integrate",
            "lagging_predicted", "lagging_pressure_update", "lagging_boundary_force_both", "lagging_positions"} <= set(c.worst)
    assert c.moved_cells >= c.ps.N // 10, (c.moved_cells, c.ps.N)


@pytest.mark.parametrize("factor,margin", [(2.0, 0.25), (0.5, -0.25)], ids=["ends", "iterates"])
def test_the_cpu_oracle_ends_its_loops_where_the_reference_does(factor, margin):
    c = _checks("block")
    c.loop_exits(factor, margin)
    assert not c.flagged(), c.worst
    assert c.exit_margin >= 100, c.exit_margin   # each decision lies far outside the error's bound


def test_the_cpu_oracle_meets_the_dt_sequence_bounds_of_the_forces():
    c = _checks("two_fluids")
    c.xsph(0.5, 0.3, dts=(DT, 2 * DT))
    c.viscosity(0.5, wcsph=2.0, dts=(DT, 2 * DT))
    assert not c.flagged(), c.worst
    c = S.Checks(_oracle, S.light(S.scene_block()))
    c.viscosity(0.5, dts=(DT, DT / 3))
    assert not c.flagged(), c.worst


@pytest.mark.parametrize("name", ["block", "two_fluids", "sixteen"])
def test_the_cpu_oracle_meets_the_iisph_warm_bounds_over_a_dt_change(name):
    c = S.Checks(lambda **kw: OracleWorld(S.R, 2.0, solver=1, **kw), S.LOOP_SCENES[name]())
    c.iisph_warm((DT, 2 * DT))
    c.iisph_warm((DT, DT / 3))
    assert not c.flagged(), c.worst
    assert {"dii_warm_dt_change", "aii_warm_dt_change", "dij_pjl_warm_dt_change", "pressure_warm_dt_change"} <= set(c.worst)


def test_the_burst_grows_the_grid_and_keeps_its_counts():
    c = S.Checks(_oracle, S.scene_burst())
    c.grid_growth()
    assert not c.flagged(), c.worst
    assert c.grown >= 1.0, c.grown


# mutant -> (scene, the checks to run, the entries that must flag it)
LOOP_MUTANTS = {
    "error_mean_over_all_fluids": ("two_fluids", "errors", {"divergence_error_read", "divergence_error"}),
    "error_drops_last_block": ("block", "errors", {"divergence_error_read", "density_error_read"}),
    "error_counts_gated": ("gate", "errors", {"divergence_error"}),
    "error_unclamped": ("block", "errors", {"density_error_read", "density_error"}),
    "div_threshold_current_inv_dt": ("block", "exits", {"divergence_exit_ends", "divergence_exit_iterates"}),
    "div_bforce_current_inv_dt": ("block", "lagging", {"lagging_boundary_force_divergence", "lagging_boundary_force_both"}),
    "xsph_current_inv_dt": ("two_fluids", "xsph", {"xsph_after_update_dt_change", "xsph_separate_dt_change"}),
    "visc_current_dt": ("light_block", "visc", {"visc_accel_1_dt_change"}),
    "positions_previous_dt": ("block", "lagging", {"lagging_positions"}),
    "vc_not_carried": ("block", "lagging", {"carried_divergence", "lagging_update"}),
    "vc_carried_unsorted": ("block", "lagging", {"carried_divergence"}),
    "fluid15_rho0_of_fluid0": ("sixteen", "stages", {"density", "divergence_sweep", "update"}),
    "iisph_previous_dt": ("block", "iisph_warm", {"dii_warm_dt_change", "aii_warm_dt_change", "dij_pjl_warm_dt_change"}),
}


def _mutant_checks(mutant):
    scene, what, must = LOOP_MUTANTS[mutant]
    sc = S.light(S.scene_block()) if scene == "light_block" else S.LOOP_SCENES[scene]()
    c = S.Checks(_oracle, sc, mutant=mutant)
    if what == "errors":
        c.loop_errors()
    elif what == "exits":
        c.loop_exits(2.0, 0.25)
        c.loop_exits(0.5, -0.25)
    elif what == "lagging":
        c.lagging_dt()
    elif what == "stages":
        c.stages()
    elif what == "iisph_warm":
        c = S.Checks(lambda **kw: OracleWorld(S.R, 2.0, solver=1, **kw), sc, mutant=mutant)
        c.iisph_warm((DT, 2 * DT))
    elif what == "xsph":
        c.xsph(0.5, 0.3, dts=(DT, 2 * DT))
    else:
        c.viscosity(0.5, dts=(DT, 2 * DT))
    return c, must


@pytest.mark.parametrize("mutant", sorted(LOOP_MUTANTS))
def test_plausible_loop_and_dt_bugs_are_caught(mutant):
    c, must = _mutant_checks(mutant)
    flagged = set(c.flagged())
    assert must <= flagged, (flagged, c.worst)


def test_every_new_mutant_has_a_case():
    assert set(LOOP_MUTANTS) <= set(S.MUTANTS)
