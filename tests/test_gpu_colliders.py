"""Collider coupling on the device (include/sph.h sph_collider_*, fluids_pipeline.rs:72-287, StaticSampling).

The engine poses the sample points itself with a fixed float32 expression, so a world whose boundaries the host rewrites
every step with the same numpy restatement must step bit for bit alike; impulses are checked against numpy sums of the
boundary forces."""
import os

import numpy as np
import pytest

from salva_b200 import BODY_DYNAMIC, BODY_FIXED, BODY_NONE, DFSPHSolver, IISPHSolver, LiquidWorld, SphError, StaticSampling, scenes
from salva_b200.liquid_world import Ball, CouplingManager, Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

F32 = np.float32
R = 0.05
DT = 0.004


def pose_points(local, rot, t):
    """world = rot @ local + t, summed left to right in float32 as k_collider_static does."""
    rot, t = np.asarray(rot, F32).reshape(3, 3), np.asarray(t, F32)
    out = np.empty_like(local)
    for a in range(3):
        out[:, a] = ((rot[a, 0] * local[:, 0] + rot[a, 1] * local[:, 1]) + rot[a, 2] * local[:, 2]) + t[a]
    return out


def local_velocity(local, linvel, angvel, com):
    """velocity_at_point(pt) at the LOCAL point (fluids_pipeline.rs:183)."""
    lv, w, c = (np.asarray(x, F32) for x in (linvel, angvel, com))
    d = local - c
    return np.stack([lv[0] + (w[1] * d[:, 2] - w[2] * d[:, 1]),
                     lv[1] + (w[2] * d[:, 0] - w[0] * d[:, 2]),
                     lv[2] + (w[0] * d[:, 1] - w[1] * d[:, 0])], axis=1).astype(F32)


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], F32)


def rot_zx(a):
    c, s = np.cos(a), np.sin(a)
    rz = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float64)
    rx = np.array([[1, 0, 0], [0, c, -s], [0, s, c]], np.float64)
    return (rz @ rx).astype(F32)


def sphere_points(radius, n=200):
    k = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * k / n)
    th = np.pi * (1 + 5 ** 0.5) * k
    return (radius * np.stack([np.cos(th) * np.sin(phi), np.cos(phi), np.sin(th) * np.sin(phi)], axis=1)).astype(F32)


def _fluid(seed=4, nx=8, ny=7, nz=8):
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, R * 0.95), R, seed, amplitude=0.3)
    vel = np.random.default_rng(seed).normal(0, 0.2, pts.shape).astype(F32)
    return pts, vel


TANK = scenes.open_tank((-R, -R, -R), (8 * 2 * R + R, 1.2, 8 * 2 * R + R), R)
TANK_OFFSET = np.array([0.25, -0.5, 0.125], F32)  # the tank's local frame sits at TANK_OFFSET (a pose test of its own)
BOX = scenes.cuboid_surface((0.15, 0.1, 0.2), R)
BALL = sphere_points(0.12)


def _states(k):
    """Per-step states of (tank, box, ball): the tank is fixed, the box a rotating dynamic body moving through the fluid,
    the ball a parentless collider far below the fluid (its samples widen the grid)."""
    tank = dict(translation=TANK_OFFSET, rotation=np.eye(3, dtype=F32), body=BODY_FIXED)
    ang = 0.3 * k
    box = dict(translation=np.array([0.4 + 0.02 * k, 0.35, 0.4], F32), rotation=rot_zx(ang), body=BODY_DYNAMIC,
               linvel=np.array([5.0, 0.0, 0.0], F32), angvel=np.array([0.0, 1.5, 2.0], F32), world_com=np.array([0.4 + 0.02 * k, 0.35, 0.4], F32))
    ball = dict(translation=np.array([0.4, -2.5 - 0.01 * k, 0.4], F32), rotation=rot_y(0.1 * k), body=BODY_NONE,
                linvel=np.array([0.0, -2.5, 0.0], F32), angvel=np.array([1.0, 0.0, 0.0], F32), world_com=np.zeros(3, F32))
    return tank, box, ball


def _host_boundary(local, st):
    p = pose_points(local, st["rotation"], st["translation"])
    if st["body"] == BODY_NONE:
        return p, np.zeros_like(p)
    return p, local_velocity(local, st.get("linvel", (0, 0, 0)), st.get("angvel", (0, 0, 0)), st.get("world_com", (0, 0, 0)))


def _make(kind, coupled):
    solver = IISPHSolver() if kind == "iisph" else DFSPHSolver(Poly6Kernel, SpikyKernel) if kind == "poly6" else DFSPHSolver()
    old = os.environ.pop("SALVA_B200_XYSUB", None)
    if kind == "rows":  # the row order of the counting sort (x / y bins of h / 2), read when a world is created
        os.environ["SALVA_B200_XYSUB"] = "2"
    try:
        w = LiquidWorld(solver, particle_radius=R)
    finally:
        os.environ.pop("SALVA_B200_XYSUB", None)
        if old is not None:
            os.environ["SALVA_B200_XYSUB"] = old
    pts, vel = _fluid()
    f = w.add_fluid(pts, velocities=vel, density0=1000.0)
    w.push_force(f, *scenes.xsph_viscosity(0.1, 0.05))
    locals_ = (TANK - TANK_OFFSET, BOX, BALL)
    if coupled:
        b = [w.add_boundary(np.zeros((0, 3), F32)) for _ in locals_]
        c = [w.register_coupling(bh, StaticSampling(l)) for bh, l in zip(b, locals_)]
    else:
        t0 = _states(0)
        b = [w.add_boundary(_host_boundary(l, s)[0], want_forces=s["body"] == BODY_DYNAMIC) for l, s in zip(locals_, t0)]
        c = None
    return w, f, b, c, locals_


def _advance(w, b, c, locals_, k):
    for j, (l, st) in enumerate(zip(locals_, _states(k))):
        if c is not None:
            w.set_collider_state(c[j], **st)
        else:
            w.write_boundary(b[j], *_host_boundary(l, st))
    w.step(DT)


@pytest.mark.parametrize("kind", ["dfsph", "rows", "iisph", "poly6"])
def test_static_colliders_match_host_posed_boundaries(kind):
    """Three StaticSampling colliders (fixed tank, dynamic rotating box, parentless ball far below the fluid) against the
    same boundaries posed by numpy and written from the host every step: fluid and boundary state bit for bit, impulses
    against numpy sums of the boundary forces."""
    dev = _make(kind, True)
    host = _make(kind, False)
    for k in range(8):
        _advance(dev[0], dev[2], dev[3], dev[4], k)
        _advance(host[0], host[2], None, host[4], k)
        wd, wh = dev[0], host[0]
        pd, vd = wd.read_fluid(dev[1])
        ph, vh = wh.read_fluid(host[1])
        assert np.array_equal(pd, ph) and np.array_equal(vd, vh), "step %d: max |dx| %g" % (k, np.abs(pd - ph).max())
        for j, (l, st) in enumerate(zip(dev[4], _states(k))):
            bp, bv = wd.read_boundary_particles(dev[2][j])
            ep, ev = _host_boundary(l, st)
            assert np.array_equal(bp, ep) and np.array_equal(bv, ev)
        vol_d, f_d = wd.read_boundary(dev[2][1])
        vol_h, f_h = wh.read_boundary(host[2][1])
        assert np.array_equal(vol_d, vol_h)
        st = _states(k)[1]
        bp, _ = wd.read_boundary_particles(dev[2][1])
        fdt = f_d.astype(np.float64) * DT
        lin = fdt.sum(axis=0)
        ang = np.cross(bp.astype(np.float64) - st["world_com"], fdt).sum(axis=0)
        got_lin, got_ang = wd.collider_impulse(dev[3][1])
        scale = np.abs(fdt).sum() + 1e-30
        assert np.abs(got_lin - lin).max() <= 1e-4 * scale
        assert np.abs(got_ang - ang).max() <= 1e-4 * scale * (1.0 + np.abs(bp - st["world_com"]).max())
        for j in (0, 2):  # fixed body: forces = None; no parent: no body to receive it
            assert not np.any(np.concatenate(wd.collider_impulse(dev[3][j])))
    assert np.abs(fdt).sum() > 0, "the box never touched the fluid"
    assert wd.stats()["grid_dims"] == wh.stats()["grid_dims"]


def test_unchanged_fixed_tank_launches_like_a_plain_boundary():
    """basic3.rs couples its tank with StaticSampling on a fixed body: with an unchanged pose the boundary's sort and
    volumes are reused, and the step launches exactly the kernels of the same tank added as a plain boundary."""
    pts, vel = _fluid(7)
    worlds = []
    for coupled in (False, True):
        w = LiquidWorld(DFSPHSolver(), particle_radius=R)
        f = w.add_fluid(pts, velocities=vel, density0=1000.0)
        if coupled:
            c = w.register_coupling(w.add_boundary(np.zeros((0, 3), F32)), StaticSampling(TANK))
            w.set_collider_state(c, body=BODY_FIXED)
        else:
            w.add_boundary(TANK)
        worlds.append((w, f))
    launches = [[], []]
    for _ in range(5):
        for i, (w, _) in enumerate(worlds):
            w.step(DT)
            launches[i].append(w.stats()["kernel_launches"])
    assert launches[0][1:] == launches[1][1:], launches
    (wa, fa), (wb, fb) = worlds
    assert np.array_equal(wa.read_fluid(fa)[0], wb.read_fluid(fb)[0])


def test_colliders_are_deterministic_across_snapshot_restore():
    """Deterministic mode: run to run, and a world restored mid-run (with its colliders registered again) continues bit
    for bit."""
    def run(steps, start=0, blob=None):
        w, f, b, c, locals_ = _make("dfsph", True)
        if blob is not None:
            w.restore(blob)
        for k in range(start, start + steps):
            _advance(w, b, c, locals_, k)
        return w, f

    half, _ = run(4)
    blob = half.snapshot()
    full, ff = run(8)
    again, fg = run(8)
    rest, fr = run(4, start=4, blob=blob)
    p_full = full.read_fluid(ff)
    for other, fo in ((again, fg), (rest, fr)):
        po = other.read_fluid(fo)
        assert np.array_equal(p_full[0], po[0]) and np.array_equal(p_full[1], po[1])


def test_unregister_and_removed_boundary():
    """unregister_coupling keeps the boundary with its last particle set (and hands it back to the host); a removed
    boundary leaves its collider inert with a zero impulse."""
    w, f, b, c, locals_ = _make("dfsph", True)
    for k in range(3):
        _advance(w, b, c, locals_, k)
    assert np.any(np.concatenate(w.collider_impulse(c[1])))
    last = w.read_boundary_particles(b[1])
    w.unregister_coupling(c[1])
    with pytest.raises(SphError):
        w.set_collider_state(c[1], body=BODY_DYNAMIC)
    w.step(DT)
    assert all(np.array_equal(x, y) for x, y in zip(w.read_boundary_particles(b[1]), last))
    w.write_boundary(b[1], last[0] + F32(0.01), last[1])  # the host owns it again
    w.step(DT)
    assert np.array_equal(w.read_boundary_particles(b[1])[0], last[0] + F32(0.01))
    # a removed boundary: inert collider
    w.set_collider_state(c[2], translation=(0.4, -2.0, 0.4), body=BODY_DYNAMIC)
    w.remove_boundary(b[2])
    w.step(DT)
    assert not np.any(np.concatenate(w.collider_impulse(c[2])))
    p, _ = w.read_fluid(f)
    assert np.isfinite(p).all()


class _Sampling:
    def __init__(self, kind, points, shape):
        self.kind, self.points, self.shape = kind, points, shape


def test_invalid_uses_are_refused():
    w, f, b, c, locals_ = _make("dfsph", True)
    _advance(w, b, c, locals_, 0)
    cases = [
        lambda: w.register_coupling(b[0], StaticSampling(BOX)),                      # already coupled
        lambda: w.write_boundary(b[1], BOX, BOX),                                    # the engine owns it
        lambda: w.set_boundary_particles(b[1], BOX),
        lambda: w.register_coupling(w.add_boundary(BOX), _Sampling(1, BOX, Ball(0.1))),  # no other sampling on the device
        lambda: w.register_coupling(w.add_boundary(BOX), StaticSampling(np.full((2, 3), np.nan, F32))),
        lambda: w.set_collider_state(c[1], translation=(np.inf, 0, 0)),
        lambda: w.set_collider_state(c[1], body=7),
        lambda: w.step_with_coupling(DT, scenes.GRAVITY, CouplingManager()),          # device and host coupling in one step
    ]
    for k, fn in enumerate(cases):
        with pytest.raises(SphError) as e:
            fn()
        assert e.value.status == 1, k

    class BadShape:
        kind, params = 9, [0.1]
    with pytest.raises(SphError):  # StaticSampling with an unknown shape attached
        w.register_coupling(w.add_boundary(BOX), _Sampling(0, BOX, BadShape()))
    _advance(w, b, c, locals_, 1)  # the refusals left the world usable
    assert np.isfinite(w.read_fluid(f)[0]).all()


class _HostColliders(CouplingManager):
    """The same StaticSampling coupling written as a host CouplingManager (coupling_manager.rs:9-28): update_boundaries
    poses the points, transmit_forces sums the impulse of the dynamic box from the boundary forces."""

    def __init__(self, b, locals_):
        self.b, self.locals, self.k, self.impulse = b, locals_, 0, None

    def update_boundaries(self, world, dt, inv_dt, h, particle_radius):
        for bh, l, st in zip(self.b, self.locals, _states(self.k)):
            world.write_boundary(bh, *_host_boundary(l, st))

    def transmit_forces(self, world, dt, inv_dt):
        st = _states(self.k)[1]
        _, f = world.read_boundary(self.b[1])
        p, _ = world.read_boundary_particles(self.b[1])
        fdt = f.astype(np.float64) * dt
        self.impulse = (fdt.sum(axis=0), np.cross(p.astype(np.float64) - st["world_com"], fdt).sum(axis=0), np.abs(fdt).sum())


def test_device_colliders_match_the_host_hook():
    """The device path against the same coupling run through sph_world_step_with_coupling."""
    dev = _make("dfsph", True)
    hook = _make("dfsph", False)
    cm = _HostColliders(hook[2], hook[4])
    for w in (dev[0], hook[0]):  # the hook re-sorts the fluid after the callback: keep error-sum order out of the comparison
        w.force_iterations(2, 3)
    h = dev[0].h
    for k in range(8):
        _advance(dev[0], dev[2], dev[3], dev[4], k)
        cm.k = k
        hook[0].step_with_coupling(DT, scenes.GRAVITY, cm)
        pd, vd = dev[0].read_fluid(dev[1])
        ph, vh = hook[0].read_fluid(hook[1])
        assert np.abs(pd - ph).max() <= 1e-5 * h and np.abs(vd - vh).max() <= 1e-4, k
        lin, ang = dev[0].collider_impulse(dev[3][1])
        scale = cm.impulse[2] + 1e-30
        assert np.abs(lin - cm.impulse[0]).max() <= 1e-4 * scale
        assert np.abs(ang - cm.impulse[1]).max() <= 1e-4 * scale


def test_refused_step_changes_nothing_and_inert_colliders_do_not_count():
    """A step refused for combining colliders with a host coupling manager applies no pending deletion; once every
    collider is unregistered or inert (its boundary removed), the host hook runs again."""
    w, f, b, c, locals_ = _make("dfsph", True)
    _advance(w, b, c, locals_, 0)
    n0 = w.num_particles(f)
    mask = np.zeros(n0, np.uint8)
    mask[:5] = 1
    w.delete_particles(f, mask)
    with pytest.raises(SphError):
        w.step_with_coupling(DT, scenes.GRAVITY, CouplingManager())
    assert w.num_particles(f) == n0
    w.unregister_coupling(c[0])
    w.unregister_coupling(c[1])
    w.remove_boundary(b[2])
    w.step_with_coupling(DT, scenes.GRAVITY, CouplingManager())
    assert w.num_particles(f) == n0 - 5
