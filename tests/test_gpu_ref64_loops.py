"""The CUDA engine's DFSPH loop errors, loop exits, lagging dt and carried state against the float64 reference
(oracle/ref64_stages.py: Checks.loop_errors, .loop_exits, .lagging_dt, .grid_growth; tests/test_ref64_loops.py checks the
CPU oracle and the mutants the bounds catch), plus the step's dt as the ABI shows it: host-callback arguments, steps too
short to run, and snapshots between steps of different length.  Each check prints the worst |err| / bound."""
import json

import numpy as np
import pytest

from oracle import ref64_stages as S
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld
from salva_b200.liquid_world import Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

DT = S.DT
F32_EPS = float(np.finfo(np.float32).eps)
K = {1: Poly6Kernel, 2: SpikyKernel}
LIBS = pytest.mark.parametrize("kd,kg", [(0, 0), (1, 2)], ids=["cubic", "poly6+spiky"])


def _gpu(kd=0, kg=0, solver=DFSPHSolver):
    def make(**kw):
        s = solver(K[kd], K[kg]) if kd else solver()
        for k, v in kw.items():
            setattr(s, k, v)
        return LiquidWorld(s, particle_radius=S.R, smoothing_factor=2.0)
    return make


def _report(c, **tags):
    print("\nREF64 %s" % json.dumps(dict(tags, worst={k: round(float(v), 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v})))
    assert not c.flagged(), c.worst


def _errors(name, kd=0, kg=0):
    c = S.Checks(_gpu(kd, kg), S.LOOP_SCENES[name](), kw=kd, kg=kg)
    c.loop_errors()
    c.loop_errors((DT, 2 * DT))
    _report(c, scene=name, check="loop_errors", kernels=[kd, kg])
    for e in ("divergence_error", "density_error"):
        assert {e, e + "_read", e + "_after_dt_change", e + "_read_after_dt_change"} <= set(c.worst)


@pytest.mark.parametrize("name", sorted(S.LOOP_SCENES))
@LIBS
def test_the_loop_errors_meet_their_bounds(name, kd, kg):
    _errors(name, kd, kg)


@pytest.mark.parametrize("name", ["block", "two_fluids", "sixteen"])
def test_the_loop_errors_meet_their_bounds_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _errors(name)


def _force(kind):
    from salva_b200 import scenes
    return scenes.xsph_viscosity(0.5, 0.0) if kind == "xsph" else scenes.akinci2013_surface_tension(1.0, 0.0)


def _launches(sc, forces):
    """Kernels launched by a step with one divergence update and no pressure update."""
    return S.run(_gpu(), sc, forces=forces, steps=[(DT, (1, 0), S.ZERO_G)])[-1]["stats"]["kernel_launches"]


@pytest.mark.parametrize("kind", ["xsph", "akinci"])
def test_the_fused_evaluations_meet_the_loop_error_bounds(kind):
    """On a single uniform-mass fluid whose boundary wants no forces (the plain block), XSPH and Akinci2013 fuse into the
    divergence evaluation after the first update (k_vel_divergence_xsph_u<1|2>), whose block partials reduce_error sums.
    The fusion shows in the launch count: there the force adds no kernel to the step, while on two fluids, where it runs
    separately, it adds some.  The loop errors are then checked as in Checks.loop_errors, fed the values read back and
    end to end, on a first step and after a dt change."""
    f = [_force(kind)]
    block, two = S.scene_block(), S.scene_two_fluids()
    assert _launches(block, f) == _launches(block, ()), "the force did not fuse into the evaluation"
    assert _launches(two, f) > _launches(two, ())
    c = S.Checks(_gpu(), block)
    c.loop_errors(forces=f)
    c.loop_errors((DT, 2 * DT), forces=f)
    _report(c, scene="block", check="loop_errors_fused_" + kind)
    for e in ("divergence_error", "density_error"):
        assert {e, e + "_read", e + "_after_dt_change", e + "_read_after_dt_change"} <= set(c.worst)


@pytest.mark.parametrize("name", ["block", "two_fluids", "sixteen"])
@LIBS
def test_the_lagging_dt_meets_every_bound(name, kd, kg):
    c = S.Checks(_gpu(kd, kg), S.LOOP_SCENES[name](), kw=kd, kg=kg)
    c.lagging_dt()
    _report(c, scene=name, check="lagging_dt", kernels=[kd, kg], moved_cells=c.moved_cells)
    assert c.moved_cells >= c.ps.N // 10


@pytest.mark.parametrize("name", ["block", "two_fluids", "sixteen"])
def test_the_lagging_dt_meets_every_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")
    c = S.Checks(_gpu(), S.LOOP_SCENES[name]())
    c.lagging_dt()
    _report(c, scene=name, check="lagging_dt_row_order")


EXITS = pytest.mark.parametrize("factor,margin", [(2.0, 0.25), (0.5, -0.25)], ids=["ends", "iterates"])


@EXITS
@LIBS
def test_the_loops_end_where_the_reference_does(factor, margin, kd, kg):
    c = S.Checks(_gpu(kd, kg), S.LOOP_SCENES["block"](), kw=kd, kg=kg)
    c.loop_exits(factor, margin)
    _report(c, scene="block", check="loop_exits", factor=factor, margin=c.exit_margin)


@EXITS
def test_the_loops_end_where_the_reference_does_in_row_order(factor, margin, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")
    c = S.Checks(_gpu(), S.LOOP_SCENES["block"]())
    c.loop_exits(factor, margin)
    _report(c, scene="block", check="loop_exits_rows", factor=factor, margin=c.exit_margin)


@pytest.mark.parametrize("name", ["block", "two_fluids", "sixteen"])
@LIBS
def test_the_iisph_warm_step_uses_the_current_dt(name, kd, kg):
    """dii, aii, dij_pjl and the pressure of a warm-started IISPH step after a dt change, all on dt_cur."""
    c = S.Checks(_gpu(kd, kg, solver=IISPHSolver), S.LOOP_SCENES[name](), kw=kd, kg=kg)
    c.iisph_warm((DT, 2 * DT))
    c.iisph_warm((DT, DT / 3))
    _report(c, scene=name, check="iisph_warm_dt_change", kernels=[kd, kg])
    assert {"dii_warm_dt_change", "aii_warm_dt_change", "dij_pjl_warm_dt_change", "pressure_warm_dt_change"} <= set(c.worst)


@LIBS
def test_the_forces_see_the_previous_dt(kd, kg):
    c = S.Checks(_gpu(kd, kg), S.LOOP_SCENES["two_fluids"](), kw=kd, kg=kg)
    c.xsph(0.5, 0.3, dts=(DT, 2 * DT))
    c.viscosity(0.5, wcsph=2.0, dts=(DT, 2 * DT))
    _report(c, scene="two_fluids", check="forces_dt_sequence", kernels=[kd, kg])
    c = S.Checks(_gpu(kd, kg), S.light(S.scene_block()), kw=kd, kg=kg)
    c.xsph(0.5, 0.0, dts=(DT, DT / 3))   # a single uniform-mass fluid: XSPH fused into the last evaluation
    c.viscosity(0.5, dts=(DT, DT / 3))
    _report(c, scene="light_block", check="forces_dt_sequence", kernels=[kd, kg])


def test_the_burst_grows_the_grid_from_the_device_bounds():
    c = S.Checks(_gpu(), S.scene_burst())
    c.grid_growth()
    _report(c, scene="burst", check="grid_growth", grown=c.grown)
    assert c.grown >= 1.0


def test_the_sixteen_fluid_scene_meets_every_pass_bound():
    c = S.Checks(_gpu(), S.scene_sixteen())
    c.stages()
    _report(c, scene="sixteen", check="stages")
    ci = S.Checks(_gpu(solver=IISPHSolver), S.scene_sixteen())
    ci.iisph_stages()
    _report(ci, scene="sixteen", check="iisph_stages")


# ---- the step's dt through the ABI ------------------------------------------------------------------------------------------
def _world(sc, calls=None, **kw):
    w = _gpu()(**kw)
    fh, bh = S.populate(w, sc)
    if calls is not None:
        w.push_host_force(fh[0], lambda dt, inv_dt, h, pos, vel, dens, acc: calls.append((dt, inv_dt)))
    return w, fh, bh


def _same_forces(fa, fb):
    """Boundary forces are summed with atomics, in an order that varies from run to run even in deterministic mode: equal
    up to the rounding of that sum, far below what a different dt or state would change."""
    assert np.abs(fa - fb).max() <= 1e-5 * np.abs(fa).max(), np.abs(fa - fb).max()
    assert np.abs(fa).max() > 0


def test_host_callbacks_see_the_previous_steps_dt():
    sc = S.LOOP_SCENES["block"]()
    calls = []
    w, _, _ = _world(sc, calls)
    dts = (DT, 2 * DT, DT / 3, DT)
    for dt in dts:
        w.step(dt)
    w.close()
    f = np.float32
    want = [(0.0, 0.0)] + [(float(f(d)), float(f(1.0) / f(d))) for d in dts[:-1]]
    assert calls == want, (calls, want)


def test_steps_too_short_to_run_only_apply_deletes():
    """dt in {0, -DT, F32_EPS} returns before the first substep (timestep_manager.rs:56-58) but after the pending deletes
    (liquid_world.rs:79-84): state, dt and inv_dt stay; the next step leaves the fluid bit-identical to a world that never
    took them."""
    sc = S.LOOP_SCENES["block"]()
    gone = np.zeros(len(sc["fluids"][0]["positions"]), np.uint8)
    gone[::7] = 1
    out = []
    for short in (True, False):
        calls = []
        w, fh, bh = _world(sc, calls)
        w.step(DT)
        P, V = w.read_fluid(fh[0])
        w.delete_particles(fh[0], gone)
        if short:
            for dt in (0.0, -DT, F32_EPS):
                w.step(dt)
            P2, V2 = w.read_fluid(fh[0])
            assert np.array_equal(P2, P[gone == 0]) and np.array_equal(V2, V[gone == 0])
        w.step(2 * DT)
        out.append((w.read_fluid(fh[0]), w.read_boundary(bh[0])[1], calls[-1]))
        w.close()
    (a, fa, ca), (b, fb, cb) = out
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    _same_forces(fa, fb)
    assert ca == cb == (float(np.float32(DT)), float(np.float32(1.0) / np.float32(DT)))


def test_a_near_zero_step_then_a_normal_one_meets_every_bound():
    """A step of nextafter(F32_EPS, 1) (inv_dt about 8.4e6) and then DT: the divergence reaction and the threshold of
    the second step carry that inv_dt."""
    c = S.Checks(_gpu(), S.LOOP_SCENES["block"]())
    eps = float(np.nextafter(np.float32(F32_EPS), np.float32(1)))
    c.lagging_dt(dts=(eps, DT), gravity=S.ZERO_G)
    c.loop_errors((eps, DT))
    _report(c, scene="block", check="near_zero_step")


def test_a_snapshot_between_steps_of_different_dt_restores_exactly():
    sc = S.LOOP_SCENES["block"]()
    calls = []
    w, fh, bh = _world(sc, calls)
    w.step(DT)
    w.step(2 * DT)
    blob = w.snapshot()
    runs = []
    for _ in range(2):
        w.step(DT / 3)
        runs.append((w.read_fluid(fh[0]), w.read_boundary(bh[0])[1], w.stats()["n_divergence_iter"], calls[-1]))
        w.restore(blob)
    w.close()
    (a, fa, na, ca), (b, fb, nb, cb) = runs
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and na == nb
    _same_forces(fa, fb)
    assert ca == cb == (float(np.float32(2 * DT)), float(np.float32(1.0) / np.float32(2 * DT)))


def test_a_dynamic_colliders_impulse_uses_the_current_dt():
    """A dynamic box coupled to the fluid over steps of DT, 2 DT, DT / 3 and DT: its linear impulse is dt_cur times the sum
    of its boundary particles' forces read back, within the float32 sum's bound (n + 2) u sum |f| dt_cur; with the
    previous step's dt it would miss that bound by far."""
    from salva_b200 import BODY_DYNAMIC, StaticSampling, scenes
    sc = S.scene_block()
    w = _gpu()()
    fh, _ = S.populate(w, sc)
    box = scenes.cuboid_surface((0.15, 0.1, 0.2), S.R)
    b = w.add_boundary(np.zeros((0, 3), np.float32))
    col = w.register_coupling(b, StaticSampling(box))
    centre = np.asarray(sc["fluids"][0]["positions"], np.float64).mean(axis=0).astype(np.float32)
    u = 2.0 ** -24
    dts = (DT, 2 * DT, DT / 3, DT)
    for k, dt in enumerate(dts):
        w.set_collider_state(col, translation=centre + np.float32(0.01 * k), body=BODY_DYNAMIC, linvel=(1.0, 0.0, 0.0),
                             angvel=(0.0, 2.0, 0.0), world_com=centre)
        w.step(dt, S.ZERO_G)
        _, f = w.read_boundary(b)
        lin, _ = w.collider_impulse(col)
        dtc = float(np.float32(dt))
        want = f.astype(np.float64).sum(axis=0) * dtc
        bound = (len(f) + 2) * u * np.abs(f.astype(np.float64)).sum(axis=0) * dtc
        assert (np.abs(lin - want) <= bound).all(), (k, lin, want, bound)
        if k and dts[k - 1] != dt:
            prev = f.astype(np.float64).sum(axis=0) * float(np.float32(dts[k - 1]))
            assert (np.abs(lin - prev) > 100 * bound).any()
    assert np.abs(f).max() > 0
    w.close()


def test_a_seventeenth_fluid_is_refused_and_changes_nothing():
    """MAX_FLUIDS = 16: adding a seventeenth fluid fails with SPH_ERR_INVALID, and the world then steps bit for bit like one
    that never tried."""
    from salva_b200.liquid_world import SphError
    sc = S.scene_sixteen()
    out = []
    for attempt in (True, False):
        w = _gpu()()
        fh, bh = S.populate(w, sc)
        if attempt:
            with pytest.raises(SphError) as e:
                w.add_fluid(np.array([[0.3, 0.9, 0.3]], np.float32))
            assert e.value.status == 1
        w.step(DT)
        w.step(2 * DT)
        out.append([w.read_fluid(f) for f in fh])
        w.close()
    for (pa, va), (pb, vb) in zip(*out):
        assert np.array_equal(pa, pb) and np.array_equal(va, vb)
