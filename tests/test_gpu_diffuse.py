"""Diffuse particles on the GPU (include/sph.h sph_world_update_diffuse, DESIGN.md section 16) against the float64
restatement in oracle/ref64_diffuse.py."""
import numpy as np
import pytest

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref64_diffuse as D  # noqa: E402
from salva_b200 import DFSPHSolver, LiquidWorld, scenes  # noqa: E402
from salva_b200.liquid_world import Poly6Kernel, SphError, SpikyKernel  # noqa: E402

F = np.float32
R = 0.05
DT = 1.0 / 200.0
FRAME = 4 * DT
G = (0.0, -9.81, 0.0)
KINDS = {"cubic": (0, 0), "poly6": (1, 2)}
VOL0 = F(0.8 * (2 * R) ** 3)
EMIT = dict(ta_min=0.5, ta_max=4.0, wc_min=0.2, wc_max=2.0, k_min=0.01, k_max=0.5, k_ta=400.0, k_wc=400.0, seed=11)


def _world(kind="cubic", deterministic=True):
    kd, kg = KINDS[kind]
    solver = DFSPHSolver(kernel_density=Poly6Kernel, kernel_gradient=SpikyKernel) if kd else None
    return LiquidWorld(solver=solver, particle_radius=R, deterministic=deterministic)


def _block(n=8, seed=3, origin=(0.0, 0.0, 0.0)):
    return scenes.jitter(scenes.block_lattice(n, n, n, R, origin=origin), R, seed)


def _shear(p, s=4.0):
    """A shear field v = (s (y - y_mid), 0, s (x - x_mid) / 2): every pair separates or approaches somewhere."""
    c = p.mean(axis=0)
    return np.stack([s * (p[:, 1] - c[1]), np.zeros(len(p)), 0.5 * s * (p[:, 0] - c[0])], 1).astype(F)


def _scene(case, kind="cubic"):
    """(world, fluids, volumes per fluid, rho0 per fluid)"""
    w = _world(kind)
    p = _block(8)
    if case == "block":
        fl = [w.add_fluid(p, velocities=np.tile(F([0.0, -2.0, 0.0]), (len(p), 1)))]
        vols = [np.full(len(p), VOL0)]
        rho = [1000.0]
    elif case == "two_fluids":
        q = _block(4, 9, origin=(0.1, 0.8, 0.1))
        v1 = (VOL0 * np.random.default_rng(5).uniform(0.6, 1.4, len(p))).astype(F)
        v2 = (VOL0 * np.random.default_rng(6).uniform(0.6, 1.4, len(q))).astype(F)
        fl = [w.add_fluid(p, velocities=_shear(p), volumes=v1), w.add_fluid(q, density0=700.0, velocities=np.tile(F([0.0, -3.0, 0.0]), (len(q), 1)),
                                                                           volumes=v2)]
        vols, rho = [v1, v2], [1000.0, 700.0]
    else:  # sheared
        fl = [w.add_fluid(p, velocities=_shear(p))]
        vols, rho = [np.full(len(p), VOL0)], [1000.0]
    side = 2 * R * 8 + R
    w.add_boundary(scenes.open_tank((-R, -R, -R), (side, 2 * side, side), R))
    return w, fl, vols, rho


def _fluid_rows(w, fl, vols, rho):
    x = np.concatenate([w.read_fluid(f)[0] for f in fl])
    v = np.concatenate([w.read_fluid(f)[1] for f in fl])
    vol = np.concatenate(vols)
    r0 = np.concatenate([np.full(w.num_particles(f), F(r)) for f, r in zip(fl, rho)])
    slots = np.concatenate([np.full(w.num_particles(f), f & 0xFFFF, np.uint32) for f in fl])
    ids = np.concatenate([w.read_ids(f) for f in fl]).astype(np.uint32)
    return x, v, vol, r0, slots, ids


def _dbg(w, fl, what):
    return np.concatenate([w.debug(f, what) for f in fl])


def _check_fluid_values(w, fl, vols, rho, kind, desc, dt, counter):
    x, v, vol, r0, slots, ids = _fluid_rows(w, fl, vols, rho)
    h = float(w.h)
    n64, ne = D.normals64(x, vol, h, KINDS[kind][1])
    ng = _dbg(w, fl, "diffuse_normal").astype(np.float64)
    good = ne < 2.0
    assert good.mean() > 0.5
    assert np.all(np.linalg.norm(ng - n64, axis=1)[good] <= ne[good]), "normals"
    P = D.potentials64(x, v, vol, r0, n64, ne, h)
    ta, wc, ek = (_dbg(w, fl, k) for k in ("diffuse_trapped_air", "diffuse_wave_crest", "diffuse_kinetic"))
    assert np.all(np.abs(ta - P["ta"]) <= P["ta_b"]), float(np.max(np.abs(ta - P["ta"]) - P["ta_b"]))
    assert np.all(np.abs(ek - P["ek"]) <= P["ek_b"])
    sure = np.abs(P["gate"] - D.GATE) > P["gate_b"]
    on = sure & (P["gate"] >= D.GATE)
    assert np.all(wc[sure & ~on] == 0.0)
    assert np.all(np.abs(wc[on] - P["kap"][on]) <= P["kap_b"][on])
    nd = _dbg(w, fl, "diffuse_count")
    want = D.counts32(ta, wc, ek, slots, ids, desc, dt, counter).astype(F)
    assert np.array_equal(nd, want)
    return nd


def _desc(w, **kw):
    d = w.diffuse_desc(**kw)
    out = {k: getattr(d, k) for k, _ in d._fields_}
    out["lo"], out["hi"] = list(d.lo), list(d.hi)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("xysub", ["1", "2"])
@pytest.mark.parametrize("case", ["block", "two_fluids", "sheared"])
def test_fluid_values_and_counts_within_the_float64_bound(case, kind, xysub, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", xysub)
    w, fl, vols, rho = _scene(case, kind)
    counter = 0
    for frame in range(3):
        if frame:  # frame 0 reads the particles as given, before the first step
            for _ in range(2):
                w.step(DT)
        w.update_diffuse(FRAME, G, **EMIT)
        nd = _check_fluid_values(w, fl, vols, rho, kind, _desc(w, **EMIT), FRAME, counter)
        counter += 1
    assert case == "block" or nd.sum() > 0
    w.close()


@pytest.mark.gpu
def test_emitted_particles_in_the_reference_order():
    w, fl, vols, rho = _scene("sheared")
    for _ in range(2):
        w.step(DT)
    every_spray = dict(EMIT, spray_below=0xFFFFFFFF, bubble_above=0xFFFFFFFF)
    st = w.update_diffuse(FRAME, (0.0, 0.0, 0.0), **every_spray)   # spray without gravity: x = x_d + dt v_d, v = v_d
    x, v, vol, r0, slots, ids = _fluid_rows(w, fl, vols, rho)
    nd = _dbg(w, fl, "diffuse_count").astype(np.int64)
    order = D.binned_order(x, slots, ids, float(w.h))
    ex, ev, bx, bv, rows = D.emit64(x[order], v[order], slots[order], ids[order], nd[order], _desc(w, **every_spray), FRAME, 0, R)
    p, pv, kind, life = w.diffuse_particles()
    assert st["emitted"] == len(ex) == len(p) > 100 and st["dropped"] == 0
    assert np.all(kind == D.SPRAY) and np.all(life == F(2.0))
    assert np.all(np.abs(pv - ev) <= bv)
    assert np.all(np.abs(p - (ex + FRAME * ev)) <= bx + FRAME * bv + 4 * D.U * np.abs(ex))
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_advection_over_several_frames(kind):
    w, fl, vols, rho = _scene("sheared", kind)
    quiet = dict(k_ta=0.0, k_wc=0.0, spray_below=6, bubble_above=20, lo=(-1.0, -0.2, -1.0), hi=(2.0, 3.0, 2.0))
    w.update_diffuse(FRAME, G, **EMIT)
    seen = set()
    for _ in range(5):
        p0, v0, k0, l0 = w.diffuse_particles()
        for _ in range(2):
            w.step(DT)
        st = w.update_diffuse(FRAME, G, **quiet)
        x, vf = np.concatenate([w.read_fluid(f)[0] for f in fl]), np.concatenate([w.read_fluid(f)[1] for f in fl])
        r = D.advect64(p0, v0, l0, x, vf, float(w.h), _desc(w, **quiet), FRAME, G, KINDS[kind][0])
        p, v, k, life = w.diffuse_particles()
        keep = r["keep"]
        assert st["emitted"] == 0 and len(p) == int(keep.sum())
        assert np.array_equal(k, r["kind"][keep].astype(np.uint8))
        assert np.all(np.abs(v - r["v"][keep]) <= r["ev"][keep] + 1e-7)
        assert np.all(np.abs(p - r["x"][keep]) <= r["ex"][keep] + 1e-7)
        assert np.allclose(life, r["life"][keep], rtol=0, atol=2e-7)
        seen |= set(np.unique(k).tolist())
    assert seen >= {D.SPRAY, D.FOAM}
    w.close()


def _twin(with_edits):
    w = _world()
    f = w.add_fluid(_block(10), velocities=_shear(_block(10)))
    side = 2 * R * 10 + R
    w.add_boundary(scenes.open_tank((-R, -R, -R), (side, 2 * side, side), R))
    if with_edits:
        w.add_sink(f, (-10.0, -10.0, -10.0), (10.0, 0.06, 10.0))
        w.add_source(f, _block(3, 4, origin=(0.3, 1.2, 0.3)), interval=4)
    return w, f


@pytest.mark.gpu
@pytest.mark.parametrize("with_edits", [False, True])
def test_updates_do_not_change_the_steps(with_edits):
    a, fa = _twin(with_edits)
    b, fb = _twin(with_edits)
    for k in range(20):
        a.step(DT)
        b.step(DT)
        if k == 7:
            for w, f in ((a, fa), (b, fb)):
                w.write_fluid(f, velocities=w.read_fluid(f)[1] * F(0.5))
        a.update_diffuse(DT, G, **EMIT)
        if k % 3 == 0:
            a.extract_surface(iso=0.6)
        assert a.snapshot() == b.snapshot()
        assert [np.array_equal(x, y) for x, y in zip(a.read_fluid(fa), b.read_fluid(fb))] == [True, True]
        assert a.step_records() == b.step_records()
    assert len(a.diffuse_particles()[0]) > 0
    if not with_edits:
        for w in (a, b):
            w.step_many(DT, 8)
        a.update_diffuse(DT, G, **EMIT)
        for w in (a, b):
            w.step_many(DT, 8)
        assert a.step_records() == b.step_records()
        assert any(r["on_device"] for r in a.step_records())
        assert a.stats()["kernel_launches"] == b.stats()["kernel_launches"]
        assert a.snapshot() == b.snapshot()
    # the surface mesh does not depend on an update before it (a step first: snapshots leave the state on the host)
    for w in (a, b):
        w.step(DT)
    b.extract_surface(iso=0.6)
    a.update_diffuse(DT, G, **EMIT)
    a.extract_surface(iso=0.6)
    for x, y in zip(a.read_surface(), b.read_surface()):
        assert np.array_equal(x, y)
    a.close()
    b.close()


@pytest.mark.gpu
def test_deterministic_and_independent_of_slot_order():
    pts = _block(9, 11)
    vel = _shear(pts)
    ids = np.arange(len(pts), dtype=np.uint32)
    perm = np.random.default_rng(2).permutation(len(pts))
    out = []
    for order in (np.arange(len(pts)), np.arange(len(pts)), perm):
        w = _world()
        f = w.add_fluid(pts[order], velocities=vel[order])
        w.set_ids(f, ids[order])
        for _ in range(3):
            w.step(DT)
            w.update_diffuse(FRAME, G, **EMIT)
        out.append(tuple(a.tobytes() for a in w.diffuse_particles()))
        w.close()
    assert len(out[0][0]) > 0
    assert out[0] == out[1] == out[2]


@pytest.mark.gpu
def test_capacity_expiry_box_and_empty_selection():
    w, fl, vols, rho = _scene("sheared")
    st = w.update_diffuse(FRAME, G, capacity=1 << 20, **dict(EMIT, seed=3))
    asked = st["emitted"]
    assert asked > 20
    w.clear_diffuse()
    assert len(w.diffuse_particles()[0]) == 0
    w2, fl2, _, _ = _scene("sheared")
    for _ in range(1):  # same counter and seed in a fresh world: the same requests, cut at capacity
        st = w2.update_diffuse(FRAME, G, capacity=17, **dict(EMIT, seed=3))
    assert st["emitted"] == 17 and st["dropped"] == asked - 17
    st = w2.update_diffuse(FRAME, G, capacity=17, **dict(EMIT, seed=3))
    assert st["emitted"] + st["spray"] + st["foam"] + st["bubble"] >= 0 and len(w2.diffuse_particles()[0]) <= 17
    # foam expiry: a lifetime shorter than one frame removes every foam particle it makes
    w3, fl3, _, _ = _scene("sheared")
    w3.update_diffuse(FRAME, G, lifetime=0.5 * FRAME, spray_below=0, bubble_above=0xFFFFFFFF, **EMIT)
    st = w3.update_diffuse(FRAME, G, lifetime=0.5 * FRAME, spray_below=0, bubble_above=0xFFFFFFFF, **EMIT)
    assert st["foam"] == 0 and st["expired"] > 0 and len(w3.diffuse_particles()[0]) == 0
    # the box: everything emitted lies outside a box far away
    st = w3.update_diffuse(FRAME, G, lo=(5.0, 5.0, 5.0), hi=(6.0, 6.0, 6.0), **EMIT)
    assert st["left_box"] == st["emitted"] > 0 and len(w3.diffuse_particles()[0]) == 0
    # empty selection, before any step, and an empty fluid
    e = _world()
    assert e.update_diffuse(FRAME, G, **EMIT)["emitted"] == 0
    f0 = e.add_fluid(np.zeros((0, 3), F))
    assert e.update_diffuse(FRAME, G, fluids=[f0], **EMIT)["emitted"] == 0
    for x in (w, w2, w3, e):
        x.close()


@pytest.mark.gpu
def test_refusals_change_nothing():
    w, fl, vols, rho = _scene("two_fluids")
    w.step(DT)
    w.update_diffuse(FRAME, G, **EMIT)
    before = [a.tobytes() for a in w.diffuse_particles()]
    snap = w.snapshot()

    def refused(dt=FRAME, g=G, fluids=None, **kw):
        with pytest.raises(SphError) as e:
            w.update_diffuse(dt, g, fluids=fluids, **dict(EMIT, **kw))
        assert e.value.status == 1
        assert [a.tobytes() for a in w.diffuse_particles()] == before
        assert w.snapshot() == snap

    refused(ta_min=float("nan"))
    refused(ta_min=4.0, ta_max=4.0)
    refused(wc_min=3.0, wc_max=2.0)
    refused(k_min=1.0, k_max=float("inf"))
    refused(k_ta=-1.0)
    refused(lifetime=0.0)
    refused(k_d=1.5)
    refused(spray_below=30, bubble_above=20)
    refused(capacity=0)
    refused(dt=0.0)
    refused(dt=float("inf"))
    refused(g=(0.0, float("nan"), 0.0))
    refused(lo=(0.0, 1.0, 0.0), hi=(1.0, 0.0, 1.0))
    refused(lo=(0.0, float("nan"), 0.0))
    refused(fluids=[fl[0], fl[0]])
    refused(fluids=[fl[0] + (7 << 16)])
    mask = np.zeros(w.num_particles(fl[0]), np.uint8)
    mask[0] = 1
    w.delete_particles(fl[0], mask)
    snap = w.snapshot()
    refused()
    seen = []

    def cb(*_):
        try:
            w.update_diffuse(FRAME, G)
            seen.append("ran")
        except SphError:
            seen.append("refused")
    w.step(DT)
    w.push_host_force(fl[1], cb)
    w.step(DT)
    assert seen == ["refused"]
    # mapped views equal the read copies
    import torch
    w.update_diffuse(FRAME, G, **EMIT)
    p, v, k, life = w.diffuse_particles()
    mp, mv, mk, ml = w.map_diffuse()
    assert np.array_equal(torch.as_tensor(mp, device="cuda").cpu().numpy(), p)
    assert np.array_equal(torch.as_tensor(mk, device="cuda").cpu().numpy(), k)
    assert np.array_equal(torch.as_tensor(ml, device="cuda").cpu().numpy(), life)
    w.close()
