"""The collider coupling on the device against the float64 reference (oracle/ref64_colliders.py), particle by particle.

Contact sampling: with the solver's iterations at zero, gravity 0 and no forces, a step is the pushes plus P += v dt, so after
each step the fluid read back is checked against the reference pushes followed by P + v dt, and every collider's samples
against the reference samples, within the stated bounds; particles at a float decision are excluded and counted.  Steps of
DT, 2 DT and DT / 3 make the lagging dt show.  StaticSampling poses and impulses are checked against their float64 sums."""
import json
import os

import numpy as np
import pytest

from oracle import ref64_colliders as C64
from salva_b200 import BODY_DYNAMIC, BODY_FIXED, DFSPHSolver, DynamicContactSampling, LiquidWorld, StaticSampling, scenes
from salva_b200.liquid_world import Ball, Capsule, Cuboid

pytestmark = pytest.mark.gpu

F = np.float32
KINDS = ["dfsph", "rows"]


def _world(kind, radius):
    old = os.environ.pop("SALVA_B200_XYSUB", None)
    if kind == "rows":  # x / y bins of h / 2, read when a world is created
        os.environ["SALVA_B200_XYSUB"] = "2"
    try:
        return LiquidWorld(DFSPHSolver(), particle_radius=radius)
    finally:
        os.environ.pop("SALVA_B200_XYSUB", None)
        if old is not None:
            os.environ["SALVA_B200_XYSUB"] = old


def _shape(kind, prm):
    return Ball(*prm) if kind == C64.BALL else Cuboid(prm) if kind == C64.CUBOID else Capsule(*prm)


def _build(sc, kind):
    """The scene's fluids and colliders; returns (world, fluids, colliders and their boundaries in slot order)."""
    R = sc["radius"]
    w = _world(kind, R)
    fl = [w.add_fluid(f["positions"], velocities=f["velocities"], density0=1000.0, memberships=f.get("memberships", 1),
                      filter=f.get("filter", 0xFFFFFFFF)) for f in sc["fluids"]]
    shapes = [DynamicContactSampling(_shape(*s)) for s in sc["shapes"]]
    if "slots" in sc:
        # fill collider slots 0..62 with StaticSampling colliders, take 63, then free 0 and 5 and take 0 again on boundary 5
        bs = [w.add_boundary(np.zeros((0, 3), F)) for _ in range(64)]
        statics = [w.register_coupling(bs[i], StaticSampling(np.zeros((0, 3), F))) for i in range(63)]
        c63 = w.register_coupling(bs[63], shapes[1])
        w.unregister_coupling(statics[0])
        w.unregister_coupling(statics[5])
        c0 = w.register_coupling(bs[5], shapes[0])
        assert (c0 & 0xFFFF, c63 & 0xFFFF) == (0, 63)
        cs, cb = [c0, c63], [bs[5], bs[63]]
    else:
        bs = []
        if sc["plain"]:
            bs.append(w.add_boundary(scenes.cuboid_surface((0.5, 0.1, 0.5), R) + np.array([0.4, -0.3, 0.4], F)))
        bs += [w.add_boundary(np.zeros((0, 3), F), memberships=2) for _ in shapes]
        cb = [bs[i] for i in sc["boundary_of_slot"]]
        cs = [w.register_coupling(b, s) for b, s in zip(cb, shapes)]  # slots in registration order, boundaries permuted
    w.force_iterations(0, 0)
    return w, fl, cs, cb


def _read(w, fl):
    parts = [w.read_fluid(f) for f in fl]
    return np.concatenate([p for p, _ in parts]), np.concatenate([v for _, v in parts])


def _contact_run(name, kind):
    sc = C64.SCENES[name]()
    w, fl, cs, cb = _build(sc, kind)
    R, h = sc["radius"], w.h
    lag, worst, excluded, candidates, firsts, branches, refs = 0.0, {}, 0, 0, None, {}, []
    for k in range(sc["steps"]):
        dt = C64.DTS[k % len(C64.DTS)]
        for c, st in zip(cs, sc["states"](k)):
            w.set_collider_state(c, **st)
        pos, vel = _read(w, fl)
        res = C64.contact64(pos, vel, C64.colliders_at(sc, k), lag, h, R)
        refs.append((pos, res))
        w.step(dt, (0.0, 0.0, 0.0))
        P, V = _read(w, fl)
        rp, rv = C64.check_fluid(res, P, V, dt)
        rs = [C64.match_samples(S, *w.read_boundary_particles(b)) for S, b in zip(res.samples, cb)]
        for key, val in (("fluid_positions", rp), ("fluid_velocities", rv), ("samples", max(rs))):
            worst[key] = max(worst.get(key, 0.0), val)
        excluded += int(res.excluded.sum())
        candidates += res.candidates
        for kd, d in res.branches.items():
            for b, n in d.items():
                branches.setdefault(kd, {}).setdefault(b, 0)
                branches[kd][b] += n
        if firsts is None:
            firsts = (res.n_samples, res.n_pushes)
        lag = dt
    cells = np.unique(np.floor(refs[0][0] / h), axis=0, return_counts=True)[1].max()
    print("\nREF64 %s" % json.dumps(dict(colliders=name, kind=kind, worst={k: round(v, 5) for k, v in worst.items()}, excluded=excluded,
                                         candidates=candidates, first_step_samples_pushes=firsts, max_cell=int(cells),
                                         branches={{1: "ball", 2: "cuboid", 3: "capsule"}[k]: {b: n for b, n in d.items() if n} for k, d in branches.items()})))
    assert max(worst.values()) <= 1.0, worst
    assert excluded <= 0.01 * candidates, (excluded, candidates)
    return sc, w, refs, firsts, branches, cells


@pytest.mark.parametrize("kind", KINDS)
def test_overlapping_colliders_meet_the_float64_bounds(kind):
    """Ball, rotated cuboid and rotated capsule whose loosened AABBs overlap, a fixed cuboid and a parentless capsule, two
    fluids with different groups, colliders registered out of boundary order: every branch of every shape reached."""
    sc, w, refs, _, br, _ = _contact_run("overlap", kind)
    res0 = refs[0][1]
    assert set(res0.processed[0].tolist()) & set(res0.processed[1].tolist()) & set(res0.processed[2].tolist())
    for kd in (C64.BALL, C64.CUBOID, C64.CAPSULE):
        for b in ("pushed", "shell", "beyond", "prediction_outside", "cell_outside", "on_surface"):
            assert br[kd][b] > 0, (kd, b)
    assert br[C64.BALL]["ball_centre"] > 0 and br[C64.CAPSULE]["capsule_axis"] > 0


@pytest.mark.parametrize("kind", KINDS)
def test_record_buffer_overflow_meets_the_float64_bounds(kind):
    """More than 4096 samples and 4096 pushes on the first step: the pass re-runs with larger buffers, and the later steps
    run on the grown ones."""
    _, _, _, firsts, _, _ = _contact_run("overflow", kind)
    assert firsts[0] > 4096 and firsts[1] > 4096, firsts


@pytest.mark.parametrize("kind", KINDS)
def test_dense_bin_and_clipped_boxes_meet_the_float64_bounds(kind):
    """A cell of more than 64 particles inside a ball; cell boxes clipped by the grid, outside it, and covering it."""
    sc, w, refs, _, _, cells = _contact_run("dense_bin_and_clipping", kind)
    assert cells > 64
    pos, res = refs[0]
    h = w.h
    lo, hi = np.floor(pos / h).min(axis=0), np.floor(pos / h).max(axis=0)
    keys = []
    for col in C64.colliders_at(sc, 0):
        ext = C64.posed_ext(col)
        t = col["translation"].astype(np.float64)
        keys.append((np.floor((t - ext - 1.5 * h) / h), np.floor((t + ext + 1.5 * h) / h)))
    assert np.any(keys[1][0] < lo) and np.all(keys[1][1] >= lo)           # clipped
    assert np.any(keys[2][0] > hi) and len(res.processed[2]) == 0        # outside
    assert np.all(keys[3][0] < lo) and np.all(keys[3][1] > hi)            # covering
    assert len(res.processed[3]) == len(pos)


@pytest.mark.parametrize("kind", KINDS)
def test_collider_slot_63_meets_the_float64_bounds(kind):
    _contact_run("high_slot", kind)


def test_static_colliders_under_rotation():
    """StaticSampling on a rotating dynamic body: the posed points and their velocities (at the LOCAL point) within the
    float64 bound; the velocity at the world point is flagged."""
    R = 0.05
    w = _world("dfsph", R)
    w.add_fluid(C64.lattice((6, 5, 6), R * 1.9, (0.0, 0.0, 0.0)), density0=1000.0)
    local = (np.random.default_rng(4).normal(0, 0.15, (400, 3))).astype(F)
    b = w.add_boundary(np.zeros((0, 3), F))
    c = w.register_coupling(b, StaticSampling(local))
    worst, mutant = 0.0, np.inf
    for k in range(4):
        st = C64._state((0.3 + 0.01 * k, 0.25, 0.3), C64.rot(0.3 * k + 0.2, -0.7, 1.1 * k), BODY_DYNAMIC, (1, -2, 0.5), (2, 1, -3),
                        (0.35, 0.2, 0.28))
        w.set_collider_state(c, **st)
        w.step(C64.DTS[k % 3])
        bp, bv = w.read_boundary_particles(b)
        x, ex, v, ev = C64.static64(local, st)
        worst = max(worst, float(C64.ratio(bp, x, ex).max()), float(C64.ratio(bv, v, ev).max()))
        _, _, vm, evm = C64.static64(local, st, mutant="world_point_velocity")
        mutant = min(mutant, float(C64.ratio(bv, vm, evm).max()))
    print("\nREF64 %s" % json.dumps(dict(colliders="static", worst=round(worst, 5), world_point_mutant=mutant)))
    assert worst <= 1.0 and mutant > 1.0


def test_impulses_meet_the_float64_bound():
    """Free-running physics under gravity over steps of DT, 2 DT, DT / 3: a submerged cuboid whose world_com lies away from
    its translation and a ball, dynamic, on adjacent boundary slots 1 and 2 with collider slots 1 and 0, and a fixed cuboid:
    each impulse within the bound of k_collider_impulse's reduction; the lagging dt and the torque about the translation
    are flagged."""
    R = 0.05
    w = _world("dfsph", R)
    w.add_fluid(C64.lattice((10, 9, 10), R * 1.9, (0.0, 0.0, 0.0), seed=2, amplitude=0.1), density0=1000.0)
    bs = [w.add_boundary(scenes.open_tank((-R, -R, -R), (10 * 1.9 * R + R, 1.2, 10 * 1.9 * R + R), R))]
    bs += [w.add_boundary(np.zeros((0, 3), F), memberships=2) for _ in range(3)]
    shapes = [(bs[2], Ball(0.12)), (bs[1], Cuboid((0.15, 0.1, 0.12))), (bs[3], Cuboid((0.1, 0.05, 0.1)))]
    cs = [w.register_coupling(b, DynamicContactSampling(s)) for b, s in shapes]
    bslot = [2, 1, 3]
    lag, worst, flagged, net = 0.0, 0.0, {"lagging_dt": 0.0, "torque_about_translation": 0.0}, []
    for k in range(6):
        dt = C64.DTS[k % 3]
        states = [C64._state((0.6, 0.35, 0.6), None, BODY_DYNAMIC, (0, -0.5, 0), (1, 0, 0.5), (0.62, 0.33, 0.6)),
                  C64._state((0.4, 0.3, 0.4), C64.rot(0.3, 0.2 + 0.05 * k, 0.1), BODY_DYNAMIC, (0.2, 0, 0), (0, 1, 0), (0.55, 0.2, 0.3)),
                  C64._state((0.9, 0.15, 0.3), C64.rot(0.1, 0.2, 0.3), BODY_FIXED)]
        for c, st in zip(cs, states):
            w.set_collider_state(c, **st)
        w.step(dt, scenes.GRAVITY)
        entries = []
        for j, ((b, _), st) in enumerate(zip(shapes, states)):
            bp, _ = w.read_boundary_particles(b)
            _, f = w.read_boundary(b)
            entries.append(dict(slot=j, bslot=bslot[j], positions=bp, forces=f, **st))
        nb = w.stats()["n_boundary_particles"]
        ref = C64.impulse64(entries, dt, lag, nb)
        for j, c in enumerate(cs):
            lin, ang = w.collider_impulse(c)
            r = max(float(C64.ratio(lin, ref[j][0], ref[j][2]).max()), float(C64.ratio(ang, ref[j][1], ref[j][3]).max()))
            worst = max(worst, r)
            if j < 2:
                f = entries[j]["forces"].astype(np.float64)
                net.append(float(np.linalg.norm(f.sum(axis=0)) / max(np.abs(f).sum(), 1e-30)))
        for m in flagged:
            mref = C64.impulse64(entries, dt, lag, nb, mutant=m)
            for j, c in enumerate(cs[:2]):
                lin, ang = w.collider_impulse(c)
                flagged[m] = max(flagged[m], float(C64.ratio(lin, mref[j][0], mref[j][2]).max()), float(C64.ratio(ang, mref[j][1], mref[j][3]).max()))
        lag = dt
    print("\nREF64 %s" % json.dumps(dict(colliders="impulse", worst=round(worst, 5), mutants=flagged, net_over_abs_sum=round(max(net), 4))))
    assert worst <= 1.0
    assert all(v > 1.0 for v in flagged.values()), flagged
