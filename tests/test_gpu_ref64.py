"""Every DFSPH and IISPH gather pass of the CUDA engine, fed its own inputs, against the float64 per-pass reference
(oracle/ref64.py), particle by particle: |gpu - ref64| <= (n_i + c_pass) u A_i + (the kernel's error term), the constants
derived in ref64.py.  One missing or corrupted contact is about a thousand times larger than that bound (tests/test_ref64.py
checks that such bugs, applied to the reference, are caught).  Each test prints the worst |err| / bound per pass and the particles excluded at float decisions."""
import json

import numpy as np
import pytest

from oracle import ref64_stages as S
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld
from salva_b200.liquid_world import Poly6Kernel, SphError, SpikyKernel, ViscosityKernel

pytestmark = pytest.mark.gpu

FORCE_SCENES = ("block", "pairs", "two_fluids")
K = {1: Poly6Kernel, 2: SpikyKernel, 3: ViscosityKernel}


def _gpu(kd=0, kg=0, backend=0):
    def make(max_divergence_iter=None):
        solver = DFSPHSolver(K[kd], K[kg]) if kd else DFSPHSolver()
        if max_divergence_iter is not None:
            solver.max_divergence_iter = max_divergence_iter
        return LiquidWorld(solver, particle_radius=S.R, smoothing_factor=2.0, gather_backend=backend)
    return make


def _check(name, kd=0, kg=0, backend=0, forces=True):
    c = S.Checks(_gpu(kd, kg, backend), S.SCENES[name](), kw=kd, kg=kg)
    c.stages()
    if forces and name in FORCE_SCENES:
        c.akinci(0.0)
        c.akinci(0.5)
        c.xsph(0.5, 0.0)
        c.xsph(0.5, 0.3)
        c.artificial(1.0, 0.0)
        c.artificial(1.0, 0.5, beta=0.3)
    print("\nREF64 %s" % json.dumps(dict(scene=name, kernels=[kd, kg], backend=backend,
                                         worst={k: round(v, 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v})))
    assert not c.flagged(), c.worst
    return c


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_every_pass_meets_its_bound(name):
    _check(name)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "volumes"])
@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_every_pass_meets_its_bound_with_generic_kernels(name, kd, kg):
    _check(name, kd, kg)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "far"])
def test_every_pass_meets_its_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _check(name)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "volumes"])
def test_every_pass_meets_its_bound_on_the_tile_backend(name):
    _check(name, backend=1)


# ---- IISPH: the density pass, dii, aii, dij_pjl, the pressure update, its density error, the velocity change and the
# boundary forces, each fed its own inputs (ref64_stages.Checks.iisph_stages) -------------------------------------------------
def _gpu_iisph(kd=0, kg=0):
    def make(min_pressure_iter=None, max_pressure_iter=None):
        solver = IISPHSolver(K[kd], K[kg]) if kd else IISPHSolver()
        if min_pressure_iter is not None:
            solver.min_pressure_iter, solver.max_pressure_iter = min_pressure_iter, max_pressure_iter
        return LiquidWorld(solver, particle_radius=S.R, smoothing_factor=2.0)
    return make


def _check_iisph(name, kd=0, kg=0):
    c = S.Checks(_gpu_iisph(kd, kg), S.SCENES[name](), kw=kd, kg=kg)
    c.iisph_stages()
    print("\nREF64 %s" % json.dumps(dict(scene=name, solver="iisph", kernels=[kd, kg],
                                         worst={k: round(v, 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v},
                                         clamped_below_above=c.clamp)))
    assert not c.flagged(), c.worst
    assert {"dii", "aii", "dij_pjl", "pressure_1", "pressure_2", "velocity", "density_error", "pressure_warm"} <= set(c.worst)
    return c


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_every_iisph_pass_meets_its_bound(name):
    _check_iisph(name)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "volumes"])
@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_every_iisph_pass_meets_its_bound_with_generic_kernels(name, kd, kg):
    _check_iisph(name, kd, kg)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "far"])
def test_every_iisph_pass_meets_its_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _check_iisph(name)


# ---- WCSPH and He2014 surface tension: WCSPH's force; He2014's colours, gradc, force and boundary reaction, each fed what its
# kernel read (ref64_stages.Checks.wcsph / .he2014) --------------------------------------------------------------------------
def _check_tension(name, kd=0, kg=0):
    c = S.Checks(_gpu(kd, kg), S.SCENES[name](), kw=kd, kg=kg)
    c.wcsph(0.5)
    for cf, cb in ((0.5, 0.0), (0.0, 0.3), (0.5, 0.3)):
        c.he2014(cf, cb)
    print("\nREF64 %s" % json.dumps(dict(scene=name, plugins="surface_tension", kernels=[kd, kg],
                                         worst={k: round(v, 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v})))
    assert not c.flagged(), c.worst
    assert {"wcsph", "he2014_color", "he2014_gradc", "he2014_force_fluid", "he2014_force_boundary", "he2014_force_both"} <= set(c.worst)
    if name == "two_fluids":
        assert "boundary_force_he2014" in c.worst
    return c


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_every_surface_tension_pass_meets_its_bound(name):
    _check_tension(name)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "volumes"])
@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_every_surface_tension_pass_meets_its_bound_with_generic_kernels(name, kd, kg):
    _check_tension(name, kd, kg)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "far"])
def test_every_surface_tension_pass_meets_its_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _check_tension(name)


# ---- Becker2009 elasticity: rest volumes, rotation, grad_tr, stress and force at the capture and after a deformation
# (ref64_stages.Checks.becker) ---------------------------------------------------------------------------------------------
def _check_becker(name, kd=0, kg=0, make=None):
    c = S.Checks(make or _gpu(kd, kg), _scene(name), kw=kd, kg=kg)
    c.becker(nonlinear=True)
    c.becker(nonlinear=False)
    print("\nREF64 %s" % json.dumps(dict(scene=name, plugins="becker2009", kernels=[kd, kg],
                                         worst={k: round(v, 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v},
                                         turn_deg=round(c.el_turn, 1), iterations=c.el_iterations)))
    assert not c.flagged(), c.worst
    assert {"el_volume", "el_deformed_nonlinear_rotation", "el_deformed_linear_force", "el_warm_nonlinear_rotation",
            "el_recaptured_volume", "el_recaptured_nonlinear_force"} <= set(c.worst)
    assert max(v for k, v in c.excluded.items() if k.endswith("rotation")) <= 0.05 * c.ps.N, c.excluded   # per stage
    return c


@pytest.mark.parametrize("name", ["block", "two_fluids", "volumes"])
def test_every_becker_pass_meets_its_bound(name):
    _check_becker(name)


@pytest.mark.parametrize("name", ["block", "two_fluids"])
def test_every_becker_pass_meets_its_bound_with_generic_kernels(name):
    _check_becker(name, 1, 2)   # Becker keeps the cubic spline in both libraries


@pytest.mark.parametrize("name", ["block", "two_fluids"])
def test_every_becker_pass_meets_its_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _check_becker(name)


@pytest.mark.parametrize("name", ["two_fluids"])
def test_every_becker_pass_meets_its_bound_under_iisph(name):
    _check_becker(name, make=_gpu_iisph())   # C5 runs Becker under IISPH


# ---- DFSPHViscosity: beta (LU residual and determinant gate), target, and the acceleration after one and two updates, with
# and without a WCSPH force before it (ref64_stages.Checks.viscosity) ---------------------------------------------------------
def _scene(name):
    return S.light(S.SCENES[name[6:]]()) if name.startswith("light_") else S.SCENES[name]()


def _check_visc(name, kd=0, kg=0):
    c = S.Checks(_gpu(kd, kg), _scene(name), kw=kd, kg=kg)
    c.viscosity(0.5)
    c.viscosity(0.5, wcsph=2.0)
    print("\nREF64 %s" % json.dumps(dict(scene=name, plugins="dfsph_viscosity", kernels=[kd, kg],
                                         worst={k: round(v, 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v}, beta_zero=c.visc_zero)))
    assert not c.flagged(), c.worst
    assert {"visc_beta", "visc_target", "visc_accel_1", "visc_accel_2", "visc_accel_2_after_wcsph"} <= set(c.worst)
    if name.startswith("light_"):
        assert c.visc_zero == 0
    return c


@pytest.mark.parametrize("name", ["light_block", "light_two_fluids", "light_volumes", "block", "tail1", "tail33"])
def test_every_viscosity_pass_meets_its_bound(name):
    _check_visc(name)


@pytest.mark.parametrize("name", ["light_block", "light_two_fluids"])
@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_every_viscosity_pass_meets_its_bound_with_generic_kernels(name, kd, kg):
    _check_visc(name, kd, kg)


@pytest.mark.parametrize("name", ["light_block", "light_two_fluids"])
def test_every_viscosity_pass_meets_its_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _check_visc(name)


def test_the_plugin_scratch_is_refused_without_its_force():
    """Selectors 12-19 refuse a fluid without the force, one whose force has not been solved yet, and one whose particles
    changed since; with a solved force they give one row of the selector's width per particle."""
    from salva_b200 import scenes
    sc = S.scene_tail(33)
    forces = {"he2014": scenes.he2014_surface_tension(0.5, 0.3), "visc": scenes.dfsph_viscosity(0.1),
              "el": scenes.becker2009_elasticity(1e5, 0.3)}
    sel = {"he2014_color": ("he2014", ()), "he2014_gradc": ("he2014", ()), "visc_beta": ("visc", (36,)),
           "visc_target": ("visc", (6,)), "el_volume0": ("el", ()), "el_rotation": ("el", (9,)), "el_grad_tr": ("el", (9,)),
           "el_stress": ("el", (6,))}
    for kind, force in forces.items():
        for stage in ("pushed", "stepped", "appended", "written"):
            w = LiquidWorld(DFSPHSolver(), particle_radius=S.R)
            (fh,), _ = S.populate(w, sc, [force])
            if stage != "pushed":
                w.step(S.DT, S.ZERO_G)
            if stage == "appended":
                w.append_particles(fh, np.array([[0.3, 0.9, 0.3]], np.float32))
            if stage == "written":   # same particles, new positions: the last solve's scratch stays readable
                w.write_fluid(fh, positions=w.read_fluid(fh)[0])
            for what, (k, shape) in sel.items():
                if k == kind and stage in ("stepped", "written"):
                    out = w.debug(fh, what)
                    assert out.shape == (33,) + shape and np.isfinite(out).all()
                else:
                    with pytest.raises(SphError):
                        w.debug(fh, what)
            w.close()


def test_the_iisph_scratch_is_refused_without_an_iisph_step():
    """A DFSPH world has no IISPH scratch, and an IISPH world has none before its first step."""
    sc = S.scene_tail(33)
    for solver, steps in ((DFSPHSolver(), 1), (IISPHSolver(), 0), (IISPHSolver(), 1)):
        w = LiquidWorld(solver, particle_radius=S.R)
        (fh,), _ = S.populate(w, sc)
        for _ in range(steps):
            w.step(S.DT, S.ZERO_G)
        for what, shape in (("dii", (33, 3)), ("aii", (33,)), ("dij_pjl", (33, 3))):
            if solver.kind == 1 and steps:
                assert w.debug(fh, what).shape == shape
            else:
                with pytest.raises(SphError):
                    w.debug(fh, what)
        w.close()
