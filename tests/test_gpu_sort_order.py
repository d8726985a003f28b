"""GPU tests of the canonical in-cell order (DESIGN.md §3) through what it decides: every f32 sum.  The cell histogram ranks a
warp's particles in input order and the in-cell sort reads its keys beside the permutation; neither may change the order the
sort ends in.  So a world that takes its particles from the host (a fresh upload, a snapshot restore, an append or delete) and
one that sorts its previous step's order must continue bit for bit alike, including worlds whose cells hold more particles than
a warp, two-fluid worlds (the key carries the fluid) and the uniform-mass path, where v* lives only in the packed records."""
import numpy as np
import pytest

from salva_b200 import DFSPHSolver, LiquidWorld, scenes

pytestmark = pytest.mark.gpu


def _scene(case, seed=11):
    r = 0.05
    rng = np.random.default_rng(seed)
    nx, ny, nz, compress = 10, 9, 8, 0.93
    forces = [scenes.xsph_viscosity(0.5, 0.2)]
    if case == "dense":  # lattice spacing r: ~(h / r)^3 = 64 particles per cell, two warps' worth
        nx, ny, nz, compress = 14, 14, 14, 0.5
    if case == "akinci":  # one uniform-mass fluid: v* only in the packed records, the fold and integration in one pass
        forces = [scenes.akinci2013_surface_tension(1.0, 0.0)]
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, r * compress), r, seed, amplitude=0.3 * compress)
    pts = pts[rng.permutation(len(pts))]  # upload order unrelated to the cells
    vel = rng.normal(0, 0.2, pts.shape).astype(np.float32)
    tank = scenes.open_tank((-r, -r, -r), (nx * 2 * r + r, 1.2, nz * 2 * r + r), r)
    fluids = [dict(positions=pts, velocities=vel, density0=1000.0, forces=list(forces))]
    if case == "two_fluids":
        up = scenes.jitter(scenes.block_lattice(nx, 4, nz, r * compress, origin=(0.0, ny * 2 * r * compress, 0.0)), r, seed + 1, amplitude=0.3)
        fluids.append(dict(positions=up, velocities=rng.normal(0, 0.2, up.shape).astype(np.float32), density0=800.0, forces=list(forces)))
    return dict(particle_radius=r, smoothing_factor=2.0, dt=0.002, gravity=scenes.GRAVITY, fluids=fluids, boundaries=[dict(positions=tank)])


def _world(sc):
    w = LiquidWorld(DFSPHSolver(), particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"], deterministic=True)
    fh, _ = scenes.populate(w, sc)
    return w, fh


def _assert_same(a, fa, b, fb):
    for k in range(len(fa)):
        pa, va = a.read_fluid(fa[k])
        pb, vb = b.read_fluid(fb[k])
        assert np.array_equal(pa, pb) and np.array_equal(va, vb)
        assert np.array_equal(a.debug(fa[k], "velocity_change"), b.debug(fb[k], "velocity_change"))


@pytest.mark.parametrize("case", ["akinci", "two_fluids", "dense"])
def test_host_round_trips_continue_bit_for_bit(case):
    """a: steps on from its own sorted order throughout.  b: restored from a's snapshot (a fresh upload in caller order).
    c: a's state written back through the host every step.  After the same appends and deletes all three agree bit for bit."""
    sc = _scene(case)
    dt = sc["dt"]
    a, fa = _world(sc)
    for _ in range(3):
        a.step(dt)
    blob = a.snapshot()
    b, fb = _world(sc)
    b.restore(blob)
    c, fc = _world(sc)
    c.restore(blob)
    for _ in range(3):
        for w, fh in ((a, fa), (b, fb), (c, fc)):
            w.step(dt)
        for k in range(len(fc)):
            c.write_fluid(fc[k], *c.read_fluid(fc[k]))
    _assert_same(a, fa, b, fb)
    _assert_same(a, fa, c, fc)

    rng = np.random.default_rng(5)
    n0 = a.num_particles(fa[0])
    mask = (rng.random(n0) < 0.1).astype(np.uint8)
    p0, _ = a.read_fluid(fa[0])
    extra = p0[rng.choice(n0, 40, replace=False)] + np.float32(0.25 * sc["particle_radius"])
    for w, fh in ((a, fa), (b, fb), (c, fc)):
        w.delete_particles(fh[0], mask)
        w.append_particles(fh[0], extra)
        for _ in range(2):
            w.step(dt)
    _assert_same(a, fa, b, fb)
    _assert_same(a, fa, c, fc)
    for w in (a, b, c):
        w.close()


def test_step_is_reproducible_run_to_run():
    """Two worlds built alike from a shuffled upload: the atomics hand out different in-cell ranks, the sums do not differ."""
    sc = _scene("dense", seed=3)
    a, fa = _world(sc)
    b, fb = _world(sc)
    for _ in range(3):
        a.step(sc["dt"])
        b.step(sc["dt"])
    _assert_same(a, fa, b, fb)
    a.close()
    b.close()
