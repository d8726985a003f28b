"""DynamicContactSampling on the device (include/sph.h SPH_SAMPLING_CONTACT, fluids_pipeline.rs:192-255).

Each step the device world is snapshotted into a twin whose host CouplingManager runs the numpy restatement
(salva_b200.contact_sampling); both step from the same state, and the samples (count, order, positions, velocities) must
be bit-identical.  With the solver's iterations at zero and no forces a step is the pushes plus pos += v dt, so the fluid
must be bit-identical too."""
import os

import numpy as np
import pytest

from salva_b200 import BODY_DYNAMIC, BODY_FIXED, BODY_NONE, DFSPHSolver, DynamicContactSampling, IISPHSolver, LiquidWorld, SphError, \
    StaticSampling, scenes
from salva_b200.contact_sampling import ContactSamplingHook, contact_sample
from salva_b200.liquid_world import Ball, Capsule, Cuboid, Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

F32 = np.float32
R = 0.05
DT = 0.004


def rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return (rz @ ry @ rx).astype(F32)


SHAPES = [(Ball(0.15), "ball"), (Cuboid((0.2, 0.08, 0.14)), "cuboid"), (Capsule(0.12, 0.07), "capsule")]


DYN3 = (BODY_DYNAMIC, BODY_DYNAMIC, BODY_DYNAMIC)


def _states(k, bodies=DYN3):
    """Per-step collider dicts in slot order: a ball and a rotated cuboid that overlap, and a rotated capsule, by default all
    on dynamic bodies with angular velocity."""
    ball = dict(translation=np.array([0.30, 0.30 - 0.01 * k, 0.30], F32), rotation=np.eye(3, dtype=F32), body=BODY_DYNAMIC,
                linvel=np.array([0.0, -1.0, 0.0], F32), angvel=np.array([0.5, 2.0, -1.0], F32), world_com=np.array([0.30, 0.30 - 0.01 * k, 0.30], F32))
    box = dict(translation=np.array([0.45, 0.28, 0.33], F32), rotation=rot(0.3 + 0.1 * k, 0.2, 0.5), body=BODY_DYNAMIC,
               linvel=np.array([0.3, 0.0, 0.1], F32), angvel=np.array([0.0, 1.5, 2.0], F32), world_com=np.array([0.40, 0.30, 0.33], F32))
    cap = dict(translation=np.array([0.20, 0.42, 0.62], F32), rotation=rot(0.7, -0.4 + 0.05 * k, 0.9), body=BODY_DYNAMIC,
               linvel=np.zeros(3, F32), angvel=np.array([-1.0, 0.0, 3.0], F32), world_com=np.array([0.20, 0.40, 0.62], F32))
    out = [ball, box, cap]
    for st, b in zip(out, bodies):
        st["body"] = b
    return out


def _coll_dicts(k, bodies=DYN3):
    return [dict(kind=s.kind, params=s.params, **st) for (s, _), st in zip(SHAPES, _states(k, bodies))]


STATIC_PTS = scenes.cuboid_surface((0.1, 0.05, 0.1), R)
STATIC_T = np.array([0.7, 0.1, 0.7], F32)
PLAIN = scenes.cuboid_surface((0.5, 0.1, 0.5), R) + np.array([0.4, -0.3, 0.4], F32)


def _fluids(seed=3):
    """Two fluids around the colliders: a jittered block with random velocities (inside, shell, beyond 1.5 h, cell in the
    box with the prediction outside and the reverse), and a second, smaller one."""
    rng = np.random.default_rng(seed)
    a = scenes.jitter(scenes.block_lattice(9, 8, 9, R * 0.95), R, seed, amplitude=0.4) + np.array([0.05, 0.08, 0.05], F32)
    va = rng.normal(0, 3.0, a.shape).astype(F32)
    b = (rng.random((300, 3)) * np.array([0.8, 0.7, 0.8]) + np.array([0.0, 0.05, 0.0])).astype(F32)
    vb = rng.normal(0, 2.0, b.shape).astype(F32)
    # one particle that, after the first step, sits one cell left of the ball's cell box with its prediction inside the
    # ball's AABB: not a candidate
    b = np.concatenate([b, np.array([[-0.2601, 0.30, 0.30]], F32)])
    vb = np.concatenate([vb, np.array([[15.0, 0.0, 0.0]], F32)])
    return (a, va), (b, vb)


def _world(kind="dfsph"):
    solver = IISPHSolver() if kind == "iisph" else DFSPHSolver(Poly6Kernel, SpikyKernel) if kind == "poly6" else DFSPHSolver()
    old = os.environ.pop("SALVA_B200_XYSUB", None)
    if kind == "rows":
        os.environ["SALVA_B200_XYSUB"] = "2"
    try:
        return LiquidWorld(solver, particle_radius=R, gather_backend=1 if kind == "tile" else 0)
    finally:
        os.environ.pop("SALVA_B200_XYSUB", None)
        if old is not None:
            os.environ["SALVA_B200_XYSUB"] = old


def _build(device, kind="dfsph", xsph=False, bodies=DYN3):
    """Fluid A does not interact with group 2 (the colliders' boundaries); fluid B interacts with everything.  The group
    filters must not change sampling."""
    w = _world(kind)
    (a, va), (b, vb) = _fluids()
    fa = w.add_fluid(a, velocities=va, density0=1000.0, memberships=1, filter=1)
    fb = w.add_fluid(b, velocities=vb, density0=1000.0)
    if xsph:
        for f in (fa, fb):
            w.push_force(f, *scenes.xsph_viscosity(0.1, 0.05))
    bs = [w.add_boundary(np.zeros((0, 3), F32), memberships=2, want_forces=b == BODY_DYNAMIC) for b in bodies]
    sb = w.add_boundary(STATIC_PTS + STATIC_T, want_forces=False)
    w.add_boundary(PLAIN)
    cs = None
    if device:
        cs = [w.register_coupling(bh, DynamicContactSampling(s)) for bh, (s, _) in zip(bs, SHAPES)]
        sc = w.register_coupling(sb, StaticSampling(STATIC_PTS))
        w.set_collider_state(sc, translation=STATIC_T, body=BODY_FIXED)
    return w, (fa, fb), bs, cs


def _set_states(w, cs, k, bodies=DYN3):
    for c, st in zip(cs, _states(k, bodies)):
        w.set_collider_state(c, **st)


def _samples(w, bs):
    return [w.read_boundary_particles(b) for b in bs]


def _lockstep(kind, xsph, gravity, iters, steps, dts, bodies=DYN3, branches=None):
    """Steps the device world and, from a snapshot of its state before each step, the twin.  `branches`: counts of the
    rule's branches on each step's input (contact_sample's), accumulated."""
    dev, fl, bs, cs = _build(True, kind, xsph, bodies)
    twin, tfl, tbs, _ = _build(False, kind, xsph, bodies)
    for w in (dev, twin):
        w.force_iterations(*iters)
    hook = ContactSamplingHook(tfl, list(zip(tbs, _coll_dicts(0, bodies))))
    lag = 0.0  # the lagging dt: 0 before the first step
    for k in range(steps):
        dt = dts[k % len(dts)]
        twin.restore(dev.snapshot())
        _set_states(dev, cs, k, bodies)
        hook.entries = list(zip(tbs, _coll_dicts(k, bodies)))
        if branches is not None:
            parts = [dev.read_fluid(f) for f in fl]
            contact_sample(np.concatenate([p for p, _ in parts]), np.concatenate([v for _, v in parts]), _coll_dicts(k, bodies), lag, dev.h, R,
                           branches)
        dev.step(dt, gravity)
        twin.step_with_coupling(dt, gravity, hook)
        lag = dt
        yield k, dev, fl, bs, cs, twin, tfl, tbs


def test_pushes_and_samples_are_bit_identical_to_numpy():
    """force_iterations(0, 0), no gravity, no forces: the fluid and every sample bit for bit, over steps of DT, 2 DT and
    DT / 3 (the lagging dt shows)."""
    sampled = 0
    branches = {}
    for k, dev, fl, bs, cs, twin, tfl, tbs in _lockstep("dfsph", False, (0.0, 0.0, 0.0), (0, 0), 9, [DT, 2 * DT, DT / 3], branches=branches):
        for f, tf in zip(fl, tfl):
            pd, vd = dev.read_fluid(f)
            pt, vt = twin.read_fluid(tf)
            assert np.array_equal(pd, pt) and np.array_equal(vd, vt), "step %d: max |dx| %g" % (k, np.abs(pd - pt).max())
        for j, ((sp, sv), (tp, tv)) in enumerate(zip(_samples(dev, bs), _samples(twin, tbs))):
            assert sp.shape == tp.shape, (k, j, sp.shape, tp.shape)
            assert np.array_equal(sp, tp) and np.array_equal(sv, tv), (k, j)
            sampled += len(sp)
        assert dev.stats()["grid_dims"] == twin.stats()["grid_dims"]
    assert sampled > 0
    # every branch of the rule was taken on the inputs the device stepped from
    for name in ("pushed", "shell", "beyond", "prediction_outside", "cell_outside"):
        assert branches.get(name, 0) > 0, (name, branches)


@pytest.mark.parametrize("kind", ["dfsph", "rows", "tile", "iisph", "poly6"])
def test_full_physics_against_the_host_hook(kind):
    """Free iterations (both worlds re-sort the fluid after the coupling, so their error sums see the same order), gravity
    and XSPH: the samples exact on each step's lockstep input, the fluid within 1e-5 h / 1e-4,
    equal grids, and impulses against numpy sums of the boundary forces."""
    for k, dev, fl, bs, cs, twin, tfl, tbs in _lockstep(kind, True, scenes.GRAVITY, (-1, -1), 6, [DT]):
        h = dev.h
        for f, tf in zip(fl, tfl):
            pd, vd = dev.read_fluid(f)
            pt, vt = twin.read_fluid(tf)
            assert np.abs(pd - pt).max() <= 1e-5 * h and np.abs(vd - vt).max() <= 1e-4, k
        for (sp, sv), (tp, tv) in zip(_samples(dev, bs), _samples(twin, tbs)):
            assert np.array_equal(sp, tp) and np.array_equal(sv, tv), k
        assert dev.stats()["grid_dims"] == twin.stats()["grid_dims"]
        for b, c, st in zip(bs, cs, _states(k)):
            bp, _ = dev.read_boundary_particles(b)
            _, f = dev.read_boundary(b)
            fdt = f.astype(np.float64) * DT
            lin = fdt.sum(axis=0)
            ang = np.cross(bp.astype(np.float64) - st["world_com"], fdt).sum(axis=0)
            got_lin, got_ang = dev.collider_impulse(c)
            scale = np.abs(fdt).sum() + 1e-30
            assert np.abs(got_lin - lin).max() <= 1e-4 * scale
            assert np.abs(got_ang - ang).max() <= 1e-4 * scale * (1.0 + np.abs(bp - st["world_com"]).max())


def test_fixed_and_parentless_bodies_sample_without_impulse():
    """A fixed body (forces dropped) and a parentless collider (zero sample velocity): the samples stay exact, and neither
    gets an impulse; the dynamic one does."""
    bodies = (BODY_FIXED, BODY_NONE, BODY_DYNAMIC)
    seen = [0, 0, 0]
    for k, dev, fl, bs, cs, twin, tfl, tbs in _lockstep("dfsph", True, scenes.GRAVITY, (-1, -1), 4, [DT], bodies=bodies):
        for j, ((sp, sv), (tp, tv)) in enumerate(zip(_samples(dev, bs), _samples(twin, tbs))):
            assert np.array_equal(sp, tp) and np.array_equal(sv, tv), (k, j)
            seen[j] += len(sp)
        assert not np.any(_samples(dev, bs)[1][1])  # no parent body: velocity 0
        for j in (0, 1):
            assert not np.any(np.concatenate(dev.collider_impulse(cs[j]))), (k, j)
    assert all(seen), seen
    assert np.any(np.concatenate(dev.collider_impulse(cs[2])))


def test_descending_ball_pushes_the_fluid_back():
    """A ball driven down into a resting block: no particle ends inside it, and the fluid pushes it back up."""
    w = LiquidWorld(DFSPHSolver(), particle_radius=R)
    pts = scenes.block_lattice(10, 6, 10, R)
    f = w.add_fluid(pts, density0=1000.0)
    w.add_boundary(scenes.open_tank((-R, -R, -R), (20 * R + R, 1.0, 20 * R + R), R))
    b = w.add_boundary(np.zeros((0, 3), F32))
    c = w.register_coupling(b, DynamicContactSampling(Ball(0.12)))
    up = 0.0
    for k in range(30):
        y = 0.75 - 0.02 * k
        w.set_collider_state(c, translation=(0.5, y, 0.5), body=BODY_DYNAMIC, linvel=(0.0, -4.0, 0.0), world_com=(0.5, y, 0.5))
        w.step(DT)
        up += float(w.collider_impulse(c)[0][1])
        p, _ = w.read_fluid(f)
        d = np.linalg.norm(p - np.array([0.5, y, 0.5], F32), axis=1)
        assert d.min() >= 0.12 - 1e-4, k
    assert up > 0


def test_snapshot_restore_unregister_remove_and_empty():
    w, fl, bs, cs = _build(True)
    for k in range(3):
        _set_states(w, cs, k)
        w.step(DT)
    blob = w.snapshot()
    ref = []
    for k in range(3, 5):
        _set_states(w, cs, k)
        w.step(DT)
    ref = [w.read_fluid(f) for f in fl], _samples(w, bs)
    w2, fl2, bs2, cs2 = _build(True)
    w2.restore(blob)
    for k in range(3, 5):
        _set_states(w2, cs2, k)
        w2.step(DT)
    got = [w2.read_fluid(f) for f in fl2], _samples(w2, bs2)
    for (a, b), (c, d) in zip(ref[0] + ref[1], got[0] + got[1]):
        assert np.array_equal(a, c) and np.array_equal(b, d)
    # unregister: the boundary keeps its last samples
    last = w.read_boundary_particles(bs[0])
    assert len(last[0]) > 0
    w.unregister_coupling(cs[0])
    w.step(DT)
    assert all(np.array_equal(x, y) for x, y in zip(w.read_boundary_particles(bs[0]), last))
    # removed boundary: inert
    w.remove_boundary(bs[1])
    w.step(DT)
    assert not np.any(np.concatenate(w.collider_impulse(cs[1])))
    # no fluid near the collider: empty boundary, zero impulse
    w.set_collider_state(cs[2], translation=(5.0, 5.0, 5.0), body=BODY_DYNAMIC)
    w.step(DT)
    assert w.read_boundary_particles(bs[2])[0].shape == (0, 3)
    assert not np.any(np.concatenate(w.collider_impulse(cs[2])))
    assert all(np.isfinite(w.read_fluid(f)[0]).all() for f in fl)


class _Sampling:
    def __init__(self, kind, points, shape):
        self.kind, self.points, self.shape = kind, points, shape


def test_refusals_leave_the_world_usable():
    w, fl, bs, cs = _build(True)
    _set_states(w, cs, 0)
    w.step(DT)
    pts = np.zeros((3, 3), F32)
    cases = [
        lambda: w.register_coupling(w.add_boundary(pts), _Sampling(1, np.zeros((0, 3), F32), None)),     # no shape
        lambda: w.register_coupling(w.add_boundary(pts), _Sampling(1, pts, Ball(0.1))),                    # points given
        lambda: w.register_coupling(w.add_boundary(pts), DynamicContactSampling(Ball(-0.1))),              # bad parameters
        lambda: w.register_coupling(w.add_boundary(pts), DynamicContactSampling(Cuboid((0.1, np.nan, 0.1)))),
        lambda: w.register_coupling(w.add_boundary(pts), DynamicContactSampling(Capsule(0.1, np.inf))),
        lambda: w.register_coupling(w.add_boundary(pts), _Sampling(2, np.zeros((0, 3), F32), Ball(0.1))),  # sampling 2
        lambda: w.write_boundary(bs[0], pts, pts),
        lambda: w.set_boundary_particles(bs[0], pts),
    ]
    for k, fn in enumerate(cases):
        with pytest.raises(SphError) as e:
            fn()
        assert e.value.status == 1, k
    _set_states(w, cs, 1)
    w.step(DT)
    assert all(np.isfinite(w.read_fluid(f)[0]).all() for f in fl)
