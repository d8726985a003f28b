"""Heightfield colliders on the device: DynamicContactSampling (k_contact_sample<true>) and particles_intersecting_shape
(k_aabb_query<true>) against the numpy restatement (salva_b200/contact_sampling.py, bit for bit) and the float64 reference
(oracle/ref64_heightfield.py, within its bounds), refusals, snapshot / restore, and the C++ example."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import ref64_colliders as rc
from oracle import ref64_heightfield as rh
from salva_b200 import BODY_DYNAMIC, BODY_FIXED, DFSPHSolver, DynamicContactSampling, LiquidWorld, SphError
from salva_b200 import contact_sampling as cs
from salva_b200.contact_sampling import ContactSamplingHook, contact_sample
from salva_b200.liquid_world import Ball, Poly6Kernel, SpikyKernel
from salva_b200.sampling import HeightField

pytestmark = pytest.mark.gpu

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
KINDS = ["dfsph", "rows", "poly6"]  # both grid orders, and the second library (poly6)
DTS = (0.004, 0.008, 0.004 / 3)


def heightfield3_heights(n=41):
    """heightfield3.rs:46-61: 3.0 on the rim, sin(i * 12 / 40) + cos(j * 12 / 40) inside."""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    x, z = (i * F(12.0) / F(n - 1)).astype(F), (j * F(12.0) / F(n - 1)).astype(F)
    h = (np.sin(x) + np.cos(z)).astype(F)
    h[[0, -1], :] = 3.0
    h[:, [0, -1]] = 3.0
    return h


def _ground():
    """heightfield3's ground (fixed body) under fluid falling onto it, with fluid below the surface and beyond the rim."""
    rng = np.random.default_rng(1)
    block = rc.lattice((24, 5, 24), 0.3, (-3.6, 1.9, -3.6), seed=1, amplitude=0.2)
    loose = (rng.uniform(-1, 1, (3000, 3)) * np.array([7.5, 2.5, 7.5]) + np.array([0, 0.5, 0])).astype(F)
    pos = np.concatenate([block, loose])
    vel = np.concatenate([np.tile(np.array([0, -4.0, 0], F), (len(block), 1)), rng.normal(0, 1, loose.shape).astype(F)])
    hf = dict(kind=rh.HEIGHTFIELD, params=(), heights=heightfield3_heights(), scale=(12.0, 1.0, 12.0))
    return dict(radius=0.15, fluids=[dict(positions=pos, velocities=vel)], colliders=[hf], boundary_of_slot=[0],
                states=lambda k: [rc._state((0, 0, 0), None, BODY_FIXED)])


def _posed():
    """A rotated, translated field on a dynamic body with angular velocity, overlapping a ball collider of the next slot,
    two fluids with group filters, the colliders registered out of boundary order."""
    rng = np.random.default_rng(9)
    H = (rng.normal(0, 0.3, (9, 13)) + 0.5).astype(F)
    a = (rng.uniform(-1, 1, (3000, 3)) * np.array([2.0, 1.0, 1.5]) + np.array([0, 0.8, 0])).astype(F)
    b = (rng.uniform(-1, 1, (800, 3)) * np.array([1.0, 0.6, 1.0]) + np.array([0.3, 0.6, 0.1])).astype(F)
    cols = [dict(kind=rh.HEIGHTFIELD, params=(), heights=H, scale=(3.0, 1.3, 2.0)), dict(kind=rc.BALL, params=(0.3,))]

    def states(k):
        return [rc._state((0.1, 0.2 - 0.01 * k, -0.1), rc.rot(0.3, 0.2 + 0.05 * k, 0.1), BODY_DYNAMIC, (0.1, -0.5, 0), (0, 1, 0.5), (0.0, 0.3, 0.0)),
                rc._state((0.5, 0.6, 0.2), None, BODY_DYNAMIC, (0, -1, 0), (1, 0, 0))]
    return dict(radius=0.05, fluids=[dict(positions=a, velocities=rng.normal(0, 1, a.shape).astype(F), memberships=1, filter=1),
                                     dict(positions=b, velocities=rng.normal(0, 1, b.shape).astype(F))],
                colliders=cols, boundary_of_slot=[1, 0], states=states)


SCENES = dict(ground=_ground, posed=_posed)


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


def _shape(col):
    return HeightField(col["heights"], col["scale"]) if col["kind"] == rh.HEIGHTFIELD else Ball(*col["params"])


def _build(sc, kind, device=True):
    w = _world(kind, sc["radius"])
    fl = [w.add_fluid(f["positions"], velocities=f["velocities"], density0=1000.0, memberships=f.get("memberships", 1),
                      filter=f.get("filter", 0xFFFFFFFF)) for f in sc["fluids"]]
    bs = [w.add_boundary(np.zeros((0, 3), F), memberships=2, want_forces=True) for _ in sc["colliders"]]
    cb = [bs[i] for i in sc["boundary_of_slot"]]
    cs = [w.register_coupling(b, DynamicContactSampling(_shape(c))) for b, c in zip(cb, sc["colliders"])] if device else None
    return w, fl, cs, cb


def _cols(sc, k):
    return [dict(c, **s) for c, s in zip(sc["colliders"], sc["states"](k))]


def _read(w, fl):
    parts = [w.read_fluid(f) for f in fl]
    return np.concatenate([p for p, _ in parts]), np.concatenate([v for _, v in parts])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_bit_identical_to_numpy_and_within_float64_bounds(scene, kind):
    """Iterations 0, no gravity, steps of DT, 2 DT, DT / 3: the fluid, every collider's samples, their counts and order are
    bit-identical to the numpy restatement run as a host hook on a twin; the heightfield pushes nothing; the samples and
    the fluid lie within the float64 bounds, with exclusions counted."""
    sc = SCENES[scene]()
    dev, fl, cs, cb = _build(sc, kind)
    twin, tfl, _, tcb = _build(sc, kind, device=False)
    for w in (dev, twin):
        w.force_iterations(0, 0)
    R, h = sc["radius"], dev.h
    lag, worst, excluded, candidates, reasons, n_hf = 0.0, {}, 0, 0, {}, 0
    for k in range(6):
        dt = DTS[k % len(DTS)]
        twin.restore(dev.snapshot())
        cols = _cols(sc, k)
        for c, st in zip(cs, sc["states"](k)):
            dev.set_collider_state(c, **st)
        pos, vel = _read(dev, fl)
        p32, _, s32 = contact_sample(pos, vel, cols, lag, h, R)
        if scene == "ground":
            assert np.array_equal(p32, pos)  # a heightfield never pushes
        res = rh.contact64(pos, vel, cols, lag, h, R)
        dev.step(dt, (0.0, 0.0, 0.0))
        twin.step_with_coupling(dt, (0.0, 0.0, 0.0), ContactSamplingHook(tfl, list(zip(tcb, cols))))
        for f, tf in zip(fl, tfl):
            pd, vd = dev.read_fluid(f)
            pt, vt = twin.read_fluid(tf)
            assert np.array_equal(pd.view(np.uint32), pt.view(np.uint32)) and np.array_equal(vd.view(np.uint32), vt.view(np.uint32)), k
        got = [dev.read_boundary_particles(b) for b in cb]
        for j, ((sp, sv), (tp, tv), (np_, nv)) in enumerate(zip(got, [twin.read_boundary_particles(b) for b in tcb], s32)):
            assert sp.shape == tp.shape == np_.shape, (k, j, sp.shape, tp.shape, np_.shape)
            assert np.array_equal(sp.view(np.uint32), tp.view(np.uint32)) and np.array_equal(sv.view(np.uint32), tv.view(np.uint32)), (k, j)
        n_hf += len(got[0][0])
        P, V = _read(dev, fl)
        rp, rv = rc.check_fluid(res, P, V, dt)
        rs = max(rc.match_samples(S, *g) for S, g in zip(res.samples, got))
        for key, val in (("fluid_positions", rp), ("fluid_velocities", rv), ("samples", rs)):
            worst[key] = max(worst.get(key, 0.0), val)
        excluded += int(res.excluded.sum())
        candidates += res.candidates + res.hf_candidates
        for key, v in res.reasons.items():
            reasons[key] = reasons.get(key, 0) + v
        lag = dt
    print("\nREF64 %s" % json.dumps(dict(scene=scene, kind=kind, worst={k: round(v, 5) for k, v in worst.items()}, excluded=excluded,
                                         candidates=candidates, reasons=reasons, heightfield_samples=n_hf)))
    assert n_hf > 1000
    assert max(worst.values()) <= 1.0, worst
    assert excluded <= 0.01 * candidates, (excluded, candidates, reasons)


def test_impulses_against_float64_sums():
    """Free-running physics with gravity: the heightfield's and the ball's impulses against float64 sums of the forces."""
    sc = _posed()
    w, fl, cs, cb = _build(sc, "dfsph")
    lag, worst = 0.0, 0.0
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
        lag = dt
    assert np.abs(entries[0]["forces"]).sum() > 0
    assert worst <= 1.0, worst


def _query_world():
    sc = _posed()
    w, fl, cs, cb = _build(sc, "dfsph", device=False)
    surf = (np.random.default_rng(4).uniform(-1, 1, (500, 3)) * np.array([1.5, 0.3, 1.0]) + np.array([0, 0.6, 0])).astype(F)
    return w, fl, w.add_boundary(surf), sc


def test_particles_intersecting_heightfield_matches_float64():
    """Fluid and boundary particles, identity and rotated poses: hit iff the float64 distance is <= particle_radius, outside
    the band where the float32 distance may fall on either side; empty before the first step, refused with edits pending."""
    w, fl, bsurf, sc = _query_world()
    H, scale = sc["colliders"][0]["heights"], sc["colliders"][0]["scale"]
    hf = HeightField(H, scale)
    assert all(len(x) == 0 for x in w.particles_intersecting_shape(hf))
    w.step(0.004, (0.0, 0.0, 0.0))
    fld = rh.field(H, scale)
    R, h = w.particle_radius, w.h
    g = cs.hf_grid(H, scale)
    checked = 0
    for t, Rot in (((0.0, 0.0, 0.0), np.eye(3, dtype=F)), ((0.1, 0.15, -0.05), rc.rot(0.2, 0.4, -0.1))):
        kinds, handles, idx = w.particles_intersecting_shape(hf, translation=t, rotation=Rot)
        got = set(zip(kinds.tolist(), handles.tolist(), idx.tolist()))
        hits = 0
        lo, hi = (np.floor(x / F(h)) for x in cs.posed_aabb(rh.HEIGHTFIELD, (), Rot, np.asarray(t, F), g))  # the cells the query visits
        for kind, handle, pts in [(0, f, w.read_fluid(f)[0]) for f in fl] + [(1, bsurf, w.read_boundary_particles(bsurf)[0])]:
            hit, decided = rh.query64(fld, pts, Rot, t, R)
            q = pts / F(h)
            hit &= np.all((np.floor(q) >= lo) & (np.floor(q) <= hi), axis=1)
            decided &= np.all(np.abs(q - np.round(q)) > 1e-4, axis=1)  # a cell key the grid may round either way
            mine = np.array([(kind, handle, i) in got for i in range(len(pts))])
            assert np.array_equal(mine[decided], hit[decided]), (kind, t)
            hits += int(hit.sum())
            checked += int(decided.sum())
            assert decided.mean() > 0.99
        assert hits > 50 and any(k == 1 for k, _, _ in got)
    assert checked > 8000
    w.append_particles(fl[0], np.array([[0.0, 3.0, 0.0]], F))
    with pytest.raises(SphError) as e:
        w.particles_intersecting_shape(hf)
    assert e.value.status == 1


def _hf_c(nrows, ncols, heights, scale):
    h = np.ascontiguousarray(heights, F)
    s = (C.c_uint32(nrows), C.c_uint32(ncols), h.ctypes.data_as(C.POINTER(C.c_float)), (C.c_float * 3)(*scale))
    from salva_b200 import _lib
    return _lib.HeightFieldC(*s), h


def test_refusals_write_nothing_and_leave_the_world_usable():
    sc = _ground()
    w, fl, cs, cb = _build(sc, "dfsph")
    w.step(0.004, (0.0, -9.81, 0.0))
    free = w.add_boundary(np.zeros((0, 3), F))
    ok = np.zeros((3, 3), F)
    bad = [(1, 3, ok[:1], (1, 1, 1)), (3, 1, ok[:1], (1, 1, 1)), (3, 3, np.array([[0, 0, 0], [0, np.nan, 0], [0, 0, 0]], F), (1, 1, 1)),
           (3, 3, ok, (1, 0, 1)), (3, 3, ok, (1, 1, -1)), (3, 3, ok, (np.inf, 1, 1))]
    L = w._L
    for nr, nc, H, s in bad:
        hf, keep = _hf_c(nr, nc, H, s)
        c = C.c_uint32(12345)
        assert L.sph_collider_register_heightfield(w._w, free, C.byref(hf), C.byref(c)) == 1 and c.value == 12345
        n = C.c_size_t(777)
        k = (C.c_uint32 * 4)(9, 9, 9, 9)
        t = (C.c_float * 3)(0, 0, 0)
        assert L.sph_world_particles_in_heightfield(w._w, C.byref(hf), t, None, k, k, k, 4, C.byref(n)) == 1
        assert n.value == 777 and list(k) == [9, 9, 9, 9]
    c = C.c_uint32(12345)
    assert L.sph_collider_register_heightfield(w._w, free, None, C.byref(c)) == 1 and c.value == 12345  # NULL heightfield
    with pytest.raises(SphError) as e:  # the ground's boundary is coupled already
        w.register_coupling(cb[0], DynamicContactSampling(HeightField(heightfield3_heights(), (12.0, 1.0, 12.0))))
    assert e.value.status == 1
    w.step(0.004, (0.0, -9.81, 0.0))
    assert np.isfinite(w.read_fluid(fl[0])[0]).all() and len(w.read_boundary_particles(cb[0])[0]) > 0


def test_snapshot_restore_and_unregister():
    """Deterministic mode: a world restored from a snapshot, with the collider registered again, continues bit for bit;
    after unregister the boundary keeps its last samples."""
    sc = _posed()
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
    last = w.read_boundary_particles(cb[0])
    assert len(last[0]) > 0
    w.unregister_coupling(cs[0])
    w.step(0.004, (0.0, -9.81, 0.0))
    assert all(np.array_equal(x, y) for x, y in zip(w.read_boundary_particles(cb[0]), last))


def test_heightfield_contact_example_runs(tmp_path):
    exe = str(tmp_path / "heightfield_contact3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "heightfield_contact3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe, "300"], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    m = re.search(r"heightfield_contact3: 3375 particles, 300 steps, first contact at step (\d+), ground samples per step (\d+)\.\.(\d+), "
                  r"(\d+) steps without samples since, (\d+) non-finite, deepest particle (\S+) below the surface", r.stdout)
    assert m, r.stdout
    first, smin, smax, empty, nan = (int(m.group(k)) for k in range(1, 6))
    print("\n" + r.stdout.strip())
    assert 0 <= first < 100 and smin > 0 and smax >= smin and empty == 0 and nan == 0
    assert np.isfinite(float(m.group(6)))
