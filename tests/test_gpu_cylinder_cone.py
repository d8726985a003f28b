"""Cylinder and cone shapes on the device: the ray sampler (k_sample_rays) against the float64 reference, DynamicContactSampling
(k_contact_sample<false, true>) bit for bit against the numpy restatement (salva_b200/contact_sampling.py) and within the
float64 bounds (oracle/ref64_revolution.py), particles_intersecting_shape (k_aabb_query<false, true>) against the reference's
decision bands, impulses, refusals, snapshot / restore and unregister."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import ref64_colliders as rc
from oracle import ref64_revolution as RV
from oracle import ref64_sampling as RS
from salva_b200 import Cone, Cylinder, DFSPHSolver, DynamicContactSampling, LiquidWorld, _lib, scenes
from salva_b200 import sampling as S
from salva_b200.contact_sampling import ContactSamplingHook
from salva_b200.liquid_world import Capsule, Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

F = np.float32
KINDS = ["dfsph", "rows", "poly6"]  # both grid orders, and the second library (poly6)
DTS = rc.DTS

SHAPES = {
    "cylinder": RS.Shape(RV.CYLINDER, [0.4, 0.27]),
    "cone": RS.Shape(RV.CONE, [0.35, 0.31]),
    "disc": RS.Shape(RV.CYLINDER, [0.0, 0.3]),
    "segment": RS.Shape(RV.CYLINDER, [0.3, 0.0]),
    "flat_cone": RS.Shape(RV.CONE, [0.0, 0.3]),
    "needle": RS.Shape(RV.CONE, [0.3, 0.0]),
}
RADII = (0.05, 0.0625, 0.037)


@pytest.fixture(scope="module", params=["lean", "kernels"])
def world(request):
    w = LiquidWorld(solver=DFSPHSolver(Poly6Kernel) if request.param == "kernels" else None, particle_radius=0.05)
    yield w
    w.close()


@pytest.mark.parametrize("volume", [False, True], ids=["surface", "volume"])
@pytest.mark.parametrize("rad", RADII)
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_sampler_matches_reference(world, name, rad, volume):
    sh = SHAPES[name]
    ref = RV.sample(sh, rad, volume)
    fn = S.shape_volume_ray_sample if volume else S.shape_surface_ray_sample
    pts = fn(world, (Cylinder if sh.kind == RV.CYLINDER else Cone)(*sh.params), rad)
    keys = RS.keys_of_points(pts, ref.origin, ref.sub)
    assert np.array_equal(pts.view(np.uint32), RS.unquantize(keys, ref.origin, ref.sub).view(np.uint32))
    assert np.all(np.diff(keys) > 0)
    missing, unexplained, und = RS.compare(keys, ref)
    assert missing == 0 and unexplained == 0, (missing, unexplained, len(ref.keys))
    print("%s %s r=%g: %d points, %d undecided keys, %d undecided ray tails" % (name, "volume" if volume else "surface", rad, len(keys), und,
                                                                               len(ref.lines)))


def _world(kind, radius):
    old = os.environ.pop("SALVA_B200_XYSUB", None)
    if kind == "rows":  # x / y bins of h / 2, read when a world is created
        os.environ["SALVA_B200_XYSUB"] = "2"
    try:
        solver = DFSPHSolver(Poly6Kernel, SpikyKernel) if kind == "poly6" else DFSPHSolver()
        return LiquidWorld(solver, particle_radius=radius)
    finally:
        os.environ.pop("SALVA_B200_XYSUB", None)
        if old is not None:
            os.environ["SALVA_B200_XYSUB"] = old


def _shape(kind, prm):
    return {RV.CYLINDER: Cylinder, RV.CONE: Cone, RV.CAPSULE: Capsule}[kind](*prm)


def _build(sc, kind, device=True):
    w = _world(kind, sc["radius"])
    fl = [w.add_fluid(f["positions"], velocities=f["velocities"], density0=1000.0, memberships=f.get("memberships", 1),
                      filter=f.get("filter", 0xFFFFFFFF)) for f in sc["fluids"]]
    bs = [w.add_boundary(scenes.cuboid_surface((0.5, 0.1, 0.5), sc["radius"]) + np.array([0.4, -0.3, 0.4], F))] if sc["plain"] else []
    bs += [w.add_boundary(np.zeros((0, 3), F), memberships=2, want_forces=True) for _ in sc["shapes"]]
    cb = [bs[i] for i in sc["boundary_of_slot"]]
    cs = [w.register_coupling(b, DynamicContactSampling(_shape(*s))) for b, s in zip(cb, sc["shapes"])] if device else None
    return w, fl, cs, cb


def _read(w, fl):
    parts = [w.read_fluid(f) for f in fl]
    return np.concatenate([p for p, _ in parts]), np.concatenate([v for _, v in parts])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scene", sorted(RV.SCENES))
def test_contact_bit_identical_to_numpy_and_within_float64_bounds(scene, kind):
    """Iterations 0, no gravity, steps of DT, 2 DT, DT / 3: the fluid and every collider's samples, counts and order are
    bit-identical to the numpy restatement run as a host hook on a twin, and lie within the float64 bounds."""
    sc = RV.SCENES[scene]()
    dev, fl, cs, cb = _build(sc, kind)
    twin, tfl, _, tcb = _build(sc, kind, device=False)
    for w in (dev, twin):
        w.force_iterations(0, 0)
    R, h = sc["radius"], dev.h
    lag, worst, excluded, candidates, reasons, nsamples = 0.0, {}, 0, 0, {}, 0
    for k in range(sc["steps"]):
        dt = DTS[k % len(DTS)]
        twin.restore(dev.snapshot())
        cols = rc.colliders_at(sc, k)
        for c, st in zip(cs, sc["states"](k)):
            dev.set_collider_state(c, **st)
        pos, vel = _read(dev, fl)
        res = RV.contact64(pos, vel, cols, lag, h, R)
        dev.step(dt, (0.0, 0.0, 0.0))
        twin.step_with_coupling(dt, (0.0, 0.0, 0.0), ContactSamplingHook(tfl, list(zip(tcb, cols))))
        for f, tf in zip(fl, tfl):
            pd, vd = dev.read_fluid(f)
            pt, vt = twin.read_fluid(tf)
            assert np.array_equal(pd.view(np.uint32), pt.view(np.uint32)) and np.array_equal(vd.view(np.uint32), vt.view(np.uint32)), k
        got = [dev.read_boundary_particles(b) for b in cb]
        for j, ((sp, sv), (tp, tv)) in enumerate(zip(got, [twin.read_boundary_particles(b) for b in tcb])):
            assert sp.shape == tp.shape, (k, j, sp.shape, tp.shape)
            assert np.array_equal(sp.view(np.uint32), tp.view(np.uint32)) and np.array_equal(sv.view(np.uint32), tv.view(np.uint32)), (k, j)
        nsamples += sum(len(g[0]) for g in got)
        P, V = _read(dev, fl)
        rp, rv = rc.check_fluid(res, P, V, dt)
        rs = max(rc.match_samples(Sm, *g) for Sm, g in zip(res.samples, got))
        for key, val in (("fluid_positions", rp), ("fluid_velocities", rv), ("samples", rs)):
            worst[key] = max(worst.get(key, 0.0), val)
        excluded += int(res.excluded.sum())
        candidates += res.candidates
        for key, v in res.reasons.items():
            reasons[key] = reasons.get(key, 0) + v
        lag = dt
    print("\nREF64 %s" % json.dumps(dict(scene=scene, kind=kind, worst={k: round(v, 5) for k, v in worst.items()}, excluded=excluded,
                                         candidates=candidates, reasons=reasons, samples=nsamples)))
    assert nsamples > 500
    assert max(worst.values()) <= 1.0, worst
    assert excluded <= 0.01 * candidates, (excluded, candidates, reasons)


def test_impulses_against_float64_sums():
    sc = RV.SCENES["posed"]()
    w, fl, cs, cb = _build(sc, "dfsph")
    lag, worst, total = 0.0, 0.0, 0.0
    for k in range(6):
        dt = DTS[k % len(DTS)]
        states = sc["states"](k)
        for c, st in zip(cs, states):
            w.set_collider_state(c, **st)
        w.step(dt, (0.0, -9.81, 0.0))
        entries = []
        for j, (b, st) in enumerate(zip(cb, states)):
            bp, _ = w.read_boundary_particles(b)
            _, f = w.read_boundary(b)
            entries.append(dict(slot=j, bslot=sc["boundary_of_slot"][j], positions=bp, forces=f, **st))
        ref = rc.impulse64(entries, dt, lag, w.stats()["n_boundary_particles"])
        for j, c in enumerate(cs):
            lin, ang = w.collider_impulse(c)
            worst = max(worst, float(rc.ratio(lin, ref[j][0], ref[j][2]).max()), float(rc.ratio(ang, ref[j][1], ref[j][3]).max()))
            total += float(np.abs(ref[j][0]).sum())
        lag = dt
    assert total > 0
    assert worst <= 1.0, worst


@pytest.mark.parametrize("kind", [RV.CYLINDER, RV.CONE])
def test_particles_intersecting_shape_matches_float64(kind):
    """Fluid and boundary particles under identity and rotated poses: hit iff the reference says so, outside its bands."""
    sc = RV.SCENES["posed"]()
    w, fl, _, _ = _build(sc, "dfsph", device=False)
    surf = (np.random.default_rng(4).uniform(0, 1, (800, 3)) * np.array([0.8, 0.7, 0.8])).astype(F)
    bsurf = w.add_boundary(surf)
    a, r = 0.15, 0.12
    shape = _shape(kind, (a, r))
    assert all(len(x) == 0 for x in w.particles_intersecting_shape(shape))
    w.force_iterations(0, 0)
    for f in fl:  # at rest, so the step leaves the particles where its cell grid puts them
        p, v = w.read_fluid(f)
        w.write_fluid(f, p, np.zeros_like(v))
    start = [w.read_fluid(f)[0] for f in fl] + [w.read_boundary_particles(bsurf)[0]]  # what the step's cell grid holds
    w.step(0.004, (0.0, 0.0, 0.0))
    R, h = w.particle_radius, w.h
    checked = 0
    for t, Rot in (((0.4, 0.35, 0.4), np.eye(3, dtype=F)), ((0.45, 0.4, 0.35), rc.rot(0.6, 0.4, -0.3))):
        kinds, handles, idx = w.particles_intersecting_shape(shape, translation=t, rotation=Rot)
        got = set(zip(kinds.tolist(), handles.tolist(), idx.tolist()))
        hits = 0
        objs = [(0, f, w.read_fluid(f)[0]) for f in fl] + [(1, bsurf, w.read_boundary_particles(bsurf)[0])]
        for (kd, handle, pts), p0 in zip(objs, start):
            hit, decided = RV.query64(kind, a, r, pts, Rot, np.asarray(t, F), h, R)
            # the cells visited hold the particles where the step's grid put them: a particle that changed cells during the
            # step, or lies at a cell face the grid may round either way, is not decided by its current cell
            q0 = p0 / F(h)
            decided &= np.all(np.floor(q0) == np.floor(pts / F(h)), axis=1) & np.all(np.abs(q0 - np.round(q0)) > 1e-4, axis=1)
            mine = np.array([(kd, handle, i) in got for i in range(len(pts))])
            assert np.array_equal(mine[decided], hit[decided]), (kd, t)
            hits += int(hit.sum())
            checked += int(decided.sum())
            assert decided.mean() > 0.9
        assert hits > 30
    assert checked > 3000


def test_refusals_write_nothing_and_leave_the_world_usable():
    sc = RV.SCENES["posed"]()
    w, fl, cs, cb = _build(sc, "dfsph")
    w.step(0.004, (0.0, -9.81, 0.0))
    free = w.add_boundary(np.zeros((0, 3), F))
    L = w._L
    for kind, p in ((5, (-0.1, 0.2)), (6, (0.1, float("nan"))), (5, (0.1, float("inf"))), (7, (0.1, 0.1)), (9, (0.1, 0.1))):
        sh = _lib.Shape()
        sh.kind = kind
        sh.p[0], sh.p[1] = p
        c = C.c_uint32(12345)
        assert L.sph_collider_register(w._w, free, 1, C.byref(sh), None, 0, C.byref(c)) == 1 and c.value == 12345
        n = C.c_size_t(777)
        k = (C.c_uint32 * 4)(9, 9, 9, 9)
        t = (C.c_float * 3)(0, 0, 0)
        assert L.sph_world_particles_in_shape(w._w, C.byref(sh), t, None, k, k, k, 4, C.byref(n)) == 1
        assert n.value == 777 and list(k) == [9, 9, 9, 9]
        out = (C.c_float * 12)(*([5.0] * 12))
        assert L.sph_world_sample_shape(w._w, 0, C.byref(sh), None, C.c_float(0.05), out, 4, C.byref(n)) == 1
        assert n.value == 777 and list(out) == [5.0] * 12
    w.step(0.004, (0.0, -9.81, 0.0))
    assert np.isfinite(w.read_fluid(fl[0])[0]).all() and sum(len(w.read_boundary_particles(b)[0]) for b in cb) > 0


def test_snapshot_restore_and_unregister():
    """Deterministic mode: a world restored from a snapshot, with the colliders registered again, continues bit for bit;
    after unregister the boundary keeps its last samples."""
    sc = RV.SCENES["posed"]()
    w, fl, cs, cb = _build(sc, "dfsph")
    for k in range(3):
        for c, st in zip(cs, sc["states"](k)):
            w.set_collider_state(c, **st)
        w.step(0.004, (0.0, -9.81, 0.0))
    blob = w.snapshot()
    w2, fl2, cs2, cb2 = _build(sc, "dfsph")
    w2.restore(blob)
    for k in range(3, 5):
        for ww, cc in ((w, cs), (w2, cs2)):
            for c, st in zip(cc, sc["states"](k)):
                ww.set_collider_state(c, **st)
            ww.step(0.004, (0.0, -9.81, 0.0))
    for a, b in zip([w.read_fluid(f) for f in fl] + [w.read_boundary_particles(b) for b in cb],
                    [w2.read_fluid(f) for f in fl2] + [w2.read_boundary_particles(b) for b in cb2]):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    j = max(range(len(cb)), key=lambda q: len(w.read_boundary_particles(cb[q])[0]))
    last = w.read_boundary_particles(cb[j])
    assert len(last[0]) > 0
    w.unregister_coupling(cs[j])
    w.step(0.004, (0.0, -9.81, 0.0))
    assert all(np.array_equal(x, y) for x, y in zip(w.read_boundary_particles(cb[j]), last))
