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
