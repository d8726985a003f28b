"""Particle sinks and sources (include/sph.h sph_fluid_add_sink / sph_fluid_add_source, DESIGN.md section 14) against a
host-driven twin.

Every step the twin does what faucet3.rs:69-105 does before the step: it reads the positions, marks the sinks' particles with
delete_particles (the same f32 box comparisons in numpy), appends each firing template with append_particles, then steps.
The world with registered sinks and sources must agree with it bit for bit after every step: positions, velocities,
velocity_changes, ids, IISPH pressures, counts, step_edits, grid_dims and the step records.  Boundary forces are float
atomics and agree to rounding."""
import numpy as np
import pytest

from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, SphError, scenes
from salva_b200.liquid_world import CouplingManager, Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

F = np.float32
R = 0.05
DT = 0.004
INF = np.inf


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == F:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def block(nx, ny, nz, origin, seed, vy=-2.0):
    p = scenes.jitter(scenes.block_lattice(nx, ny, nz, R * 0.95, origin=origin), R, seed, amplitude=0.3)
    v = np.random.default_rng(seed).normal(0, 0.1, p.shape).astype(F)
    v[:, 1] += F(vy)
    return p, v


def sheet(n, y, x0=0.1, z0=0.1, vy=-1.0):
    g = np.arange(n, dtype=F) * F(2 * R)
    p = np.stack(np.meshgrid(g + F(x0), np.array([y], F), g + F(z0), indexing="ij"), -1).reshape(-1, 3).astype(F)
    v = np.zeros_like(p)
    v[:, 1] = vy
    return p, v


TANK = scenes.open_tank((-R, -0.6, -R), (1.0, 0.8, 1.0), R)


def scene(name):
    """Fluids (positions, velocities, volumes, density0, memberships, filter, forces), boundaries, solver, sinks
    (fluid, lo, hi, outside) and sources (fluid, positions, velocities, interval); make() also takes a particle_radius
    (default R)."""
    p, v = block(6, 6, 6, (0.1, 0.0, 0.1), 3)
    fl = dict(positions=p, velocities=v, density0=1000.0, forces=[])
    sc = dict(solver=DFSPHSolver(), fluids=[fl], boundaries=[TANK], sinks=[], sources=[], forces_wanted=False)
    drain = (0, (-INF, -INF, -INF), (INF, 0.05, INF), 0)
    s1 = sheet(4, 0.75)
    sc["sinks"] = [drain]
    sc["sources"] = [(0, s1[0], s1[1], 3)]
    if name == "quiet":
        sc["sinks"].append((0, (-0.2, -1.0, -0.2), (1.2, 2.0, 1.2), 1))  # a domain sink
    elif name == "xsph":
        fl["forces"] = [scenes.xsph_viscosity(0.5, 0.0)]
    elif name == "akinci":
        fl["forces"] = [scenes.akinci2013_surface_tension(1.0, 0.0)]
        sc["boundaries"] = []
    elif name == "two_fluids":
        p2, v2 = block(5, 3, 5, (0.4, 0.4, 0.4), 7)
        sc["fluids"].append(dict(positions=p2, velocities=v2, density0=800.0, memberships=2, filter=0xFFFFFFFF ^ 2,
                                 forces=[scenes.artificial_viscosity(1.0, 0.0)]))
        sc["sinks"].append((1, (-INF, -INF, -INF), (INF, 0.3, INF), 0))
        sc["sources"] = [(0, s1[0], s1[1], 2), (1, s1[0][:5] + F(0.3), None, 4)]
        sc["forces_wanted"] = True
    elif name == "iisph_becker":
        sc["solver"] = IISPHSolver()
        fl["forces"] = [scenes.becker2009_elasticity(1.0e5, 0.3)]
    elif name == "dfsph_viscosity":
        fl["positions"], fl["velocities"] = block(6, 6, 6, (0.1, 0.0, 0.1), 3, vy=0.0)
        # one viscosity iteration per step at a small coefficient: the reference's loop amplifies its error on a free
        # surface (tests/test_gpu_parity.py::test_dfsph_viscosity_row_a16), and larger settings blow this scene up
        fl["forces"] = [scenes.dfsph_viscosity(0.05, 1, 1, 0.01)]
        sc["sinks"] = [(0, (-INF, -INF, -INF), (INF, 0.12, INF), 0)]
        s2 = sheet(4, 0.575, x0=0.15, z0=0.15, vy=0.0)  # onto the block's top layer: no particle without neighbours
        sc["sources"] = [(0, s2[0], s2[1], 8)]
    elif name == "volumes":
        fl["volumes"] = (R ** 3 * 6.4 * np.random.default_rng(5).uniform(0.95, 1.05, len(p))).astype(F)
        fl["forces"] = [scenes.xsph_viscosity(0.2, 0.0)]
    elif name == "ball":  # faucet3's ball, sampled on its surface; no tank
        th = np.random.default_rng(2).uniform(0, 2 * np.pi, 300)
        ph = np.arccos(np.random.default_rng(3).uniform(-1, 1, 300))
        ball = np.stack([np.sin(ph) * np.cos(th), np.cos(ph), np.sin(ph) * np.sin(th)], -1) * 0.15 + np.array([0.25, -0.3, 0.25])
        sc["boundaries"] = [ball.astype(F)]
        sc["sinks"] = [(0, (-INF, -INF, -INF), (INF, -0.2, INF), 0)]
    elif name == "poly6":
        sc["solver"] = DFSPHSolver(kernel_density=Poly6Kernel, kernel_gradient=SpikyKernel)
    else:
        raise ValueError(name)
    return sc


def make(sc):
    w = LiquidWorld(solver=sc["solver"], particle_radius=sc.get("particle_radius", R), smoothing_factor=2.0)
    fh = []
    for f in sc["fluids"]:
        h = w.add_fluid(f["positions"], density0=f["density0"], velocities=f["velocities"], volumes=f.get("volumes"),
                        memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF))
        for kind, params in f["forces"]:
            w.push_force(h, kind, params)
        fh.append(h)
    bh = [w.add_boundary(b, want_forces=sc["forces_wanted"]) for b in sc["boundaries"]]
    return w, fh, bh


class Pair:
    """The world under test (sinks and sources registered) and its host-driven twin, stepped together."""

    def __init__(self, sc):
        self.sc = sc
        self.a, self.fa, self.ba = make(sc)
        self.b, self.fb, self.bb = make(sc)
        self.sinks, self.sources = [], []  # twin side: (fluid index, lo, hi, outside, handle) / (fluid, p, v, interval, age, handle)
        for s in sc["sinks"]:
            self.add_sink(*s)
        for s in sc["sources"]:
            self.add_source(*s)

    def add_sink(self, fi, lo, hi, outside):
        h = self.a.add_sink(self.fa[fi], lo, hi, outside=bool(outside))
        self.sinks.append([fi, np.asarray(lo, F), np.asarray(hi, F), outside, h])
        return h

    def add_source(self, fi, p, v, interval):
        h = self.a.add_source(self.fa[fi], p, v, interval)
        self.sources.append([fi, p, v, interval, 0, h])
        return h

    def remove_sink(self, h):
        self.a.remove_sink(h)
        self.sinks = [s for s in self.sinks if s[4] != h]

    def remove_source(self, h):
        self.a.remove_source(h)
        self.sources = [s for s in self.sources if s[5] != h]

    def twin_edits(self):
        want = []
        for fi, hb in enumerate(self.fb):
            if hb is None:
                want.append(None)
                continue
            p, _ = self.b.read_fluid(hb)
            mask = np.zeros(len(p), bool)
            for sfi, lo, hi, outside, _h in self.sinks:
                if sfi != fi:
                    continue
                inb = np.all((lo <= p) & (p < hi), axis=1)
                mask |= ~inb if outside else inb
            if mask.any():
                self.b.delete_particles(hb, mask)
            emitted = 0
            for src in self.sources:
                if src[0] == fi and src[4] % src[3] == 0:
                    self.b.append_particles(hb, src[1], src[2])
                    emitted += len(src[1])
            want.append((int(mask.sum()), emitted))
        for src in self.sources:
            src[4] += 1
        return want

    def step(self, dt=DT, coupling=None):
        want = self.twin_edits()
        errors = []
        for w in (self.a, self.b):
            try:
                if coupling:
                    w.step_with_coupling(dt, scenes.GRAVITY, coupling)
                else:
                    w.step(dt)
                errors.append(None)
            except SphError as e:
                errors.append(str(e))
        assert errors[0] == errors[1]
        if errors[0]:
            raise SphError(1, errors[0])
        for fi, w in enumerate(want):
            if w is not None:
                assert self.a.step_edits(self.fa[fi]) == w
        self.check()
        return want

    def check(self, debug=()):
        a, b = self.a, self.b
        iisph = isinstance(self.sc["solver"], IISPHSolver)
        for x, y in zip(self.fa, self.fb):
            if x is None:
                continue
            assert a.num_particles(x) == b.num_particles(y)
            pa, va = a.read_fluid(x)
            pb, vb = b.read_fluid(y)
            assert same(pa, pb) and same(va, vb)
            assert same(a.debug(x, "velocity_change"), b.debug(y, "velocity_change"))
            assert same(a.read_ids(x), b.read_ids(y))
            if iisph:
                assert same(a.debug(x, "pressure"), b.debug(y, "pressure"))
            for what in debug:
                ea = eb = None
                try:
                    ra = a.debug(x, what)
                except SphError as e:
                    ea = e
                try:
                    rb = b.debug(y, what)
                except SphError as e:
                    eb = e
                assert (ea is None) == (eb is None), what
                if ea is None:
                    assert same(ra, rb), what
        sa, sb = a.stats(), b.stats()
        for k in ("grid_dims", "n_fluid_particles", "n_boundary_particles", "n_divergence_iter", "n_pressure_iter", "n_divergence_eval",
                  "n_pressure_eval", "max_neighbors", "n_contacts"):
            assert sa[k] == sb[k], k
        assert a.step_records() == b.step_records()
        if self.sc["forces_wanted"]:
            for x, y in zip(self.ba, self.bb):
                va, fa = a.read_boundary(x)
                vb, fb = b.read_boundary(y)
                assert same(va, vb)
                np.testing.assert_allclose(fa, fb, rtol=1e-5, atol=1e-6 * max(1.0, float(np.abs(fb).max(initial=0.0))))


@pytest.mark.parametrize("xysub", ["1", "2"])
@pytest.mark.parametrize("name", ["quiet", "xsph", "akinci", "two_fluids", "iisph_becker", "dfsph_viscosity", "volumes", "ball", "poly6"])
def test_matches_the_host_driven_twin(name, xysub, monkeypatch):
    if xysub == "2" and name not in ("xsph", "two_fluids", "iisph_becker"):
        pytest.skip("row order: three scenes")
    monkeypatch.setenv("SALVA_B200_XYSUB", xysub)
    sc = scene(name)
    P = Pair(sc)
    dbg = {"iisph_becker": ("el_volume0", "el_rotation"), "dfsph_viscosity": ("visc_target",)}.get(name, ())
    removed = emitted = 0
    for k in range(24):
        want = P.step()
        P.check(debug=dbg)
        removed += want[0][0]
        emitted += want[0][1]
    assert removed > 0 and emitted > 0  # both kinds acted


def test_coupling_step():
    class Push(CouplingManager):
        def update_boundaries(self, world, dt, inv_dt, h, r):
            pass

    P = Pair(scene("xsph"))
    for _ in range(10):
        P.step(coupling=Push())


def test_emptied_fluid_is_refilled_and_ids_count_on():
    sc = scene("quiet")
    sc["sinks"], sc["sources"] = [], []
    P = Pair(sc)
    h = P.add_sink(0, (-INF, -INF, -INF), (INF, INF, INF), 0)  # everything
    P.step()
    assert P.a.num_particles(P.fa[0]) == 0
    P.remove_sink(h)
    s = sheet(3, 0.5)
    P.add_source(0, s[0], s[1], 2)
    for _ in range(5):
        P.step()
    assert P.a.num_particles(P.fa[0]) == 27
    assert np.array_equal(P.a.read_ids(P.fa[0]), np.arange(27))  # an empty fluid numbers from 0, as sph_fluid_append does


def test_marks_sink_and_source_in_one_step():
    sc = scene("xsph")
    P = Pair(sc)
    for _ in range(3):
        P.step()
    for w, f in ((P.a, P.fa[0]), (P.b, P.fb[0])):
        ids = w.read_ids(f)
        w.delete_particles(f, ids == ids.max())  # the largest id is marked in the step the source fires again
    assert P.step()[0][1] > 0
    P.step()


def test_host_append_between_steps_then_source():
    P = Pair(scene("xsph"))
    P.step()
    extra = sheet(2, 0.6, x0=0.3)[0]
    for w, f in ((P.a, P.fa[0]), (P.b, P.fb[0])):
        w.append_particles(f, extra)
    for _ in range(4):
        P.step()


def test_zero_dt_steps_count_and_edit():
    P = Pair(scene("xsph"))
    P.step(0.0)
    P.step(0.0)
    P.step()
    P.step(0.0)
    P.step()


def test_box_edges_and_infinite_bounds():
    sc = scene("quiet")
    sc["sinks"], sc["sources"] = [], []
    P = Pair(sc)
    p, _ = P.a.read_fluid(P.fa[0])
    y = np.unique(p[:, 1])
    lo, hi = y[3], y[40]  # particles exactly on lo are removed, exactly on hi are kept
    P.add_sink(0, (-INF, lo, -INF), (INF, hi, INF), 0)
    P.step()
    P.add_sink(0, (p[:, 0].min(), -INF, -INF), (INF, INF, INF), 1)
    for _ in range(3):
        P.step()


def test_domain_sink_removes_a_non_finite_particle():
    sc = scene("quiet")
    sc["sinks"], sc["sources"] = [], []
    P = Pair(sc)
    P.add_sink(0, (-INF, -INF, -INF), (INF, INF, INF), 1)  # removes only what is in no box: non-finite positions
    for w, f in ((P.a, P.fa[0]), (P.b, P.fb[0])):
        p, v = w.read_fluid(f)
        p[7] = (np.nan, 0.1, 0.1)
        p[9] = (0.1, np.inf, 0.1)
        w.write_fluid(f, p, v)
    P.step()
    assert P.a.step_edits(P.fa[0]) == (2, 0)
    P.step()


def test_interval_and_a_source_registered_mid_run():
    sc = scene("xsph")
    sc["sinks"], sc["sources"] = [], []
    P = Pair(sc)
    s = sheet(2, 0.7)
    P.add_source(0, s[0], None, 3)
    fired = [P.step()[0][1] > 0 for _ in range(8)]
    assert fired == [True, False, False, True, False, False, True, False]  # steps 1, 4, 7
    P.add_source(0, s[0] + F(0.2), s[1], 2)
    for _ in range(5):
        P.step()


def test_remove_source_sink_and_fluid():
    sc = scene("two_fluids")
    P = Pair(sc)
    P.step()
    gone_source, gone_sink = P.sources[0][5], P.sinks[0][4]
    P.remove_source(gone_source)
    P.remove_sink(gone_sink)
    P.step()
    P.step()
    with pytest.raises(SphError):
        P.a.remove_sink(gone_sink)
    with pytest.raises(SphError):
        P.a.remove_source(gone_source)
    fluid0_sink = P.add_sink(0, (-INF, -INF, -INF), (INF, -5.0, INF), 0)
    for w, f in ((P.a, P.fa[0]), (P.b, P.fb[0])):
        w.remove_fluid(f)
    P.sinks = [s for s in P.sinks if s[0] != 0]
    P.sources = [s for s in P.sources if s[0] != 0]
    P.fa[0] = P.fb[0] = None
    for _ in range(3):
        P.step()
    with pytest.raises(SphError):
        P.a.remove_sink(fluid0_sink)  # remove_fluid removed it


def test_snapshot_restore_keeps_registrations_and_counts():
    P = Pair(scene("xsph"))
    for _ in range(4):
        P.step()
    blob_a, blob_b = P.a.snapshot(), P.b.snapshot()
    for _ in range(3):
        P.step()
    P.a.restore(blob_a)
    P.b.restore(blob_b)
    for _ in range(4):  # the source's step count runs on from 7
        P.step()


def test_refusals_change_nothing():
    P = Pair(scene("xsph"))
    P.step()
    a, f = P.a, P.fa[0]

    def state():
        p, v = a.read_fluid(f)
        return p, v, a.read_ids(f), a.debug(f, "velocity_change")

    s0 = state()
    for lo, hi, outside in (((np.nan, 0, 0), (1, 1, 1), 0), ((0, 2, 0), (1, 1, 1), 0), ((0, 0, 0), (1, 1, 1), 2)):
        with pytest.raises(SphError):
            a.add_sink(f, lo, hi, outside)
    with pytest.raises(SphError):
        a.add_source(f, sheet(2, 0.5)[0], None, 0)
    with pytest.raises(SphError):
        a.add_source(f, np.zeros((0, 3), F), None, 1)
    with pytest.raises(SphError):
        a.remove_source(P.sources[0][5] + (1 << 16))  # stale generation
    with pytest.raises(SphError):
        a.step_many(DT, 2)
    assert all(same(x, y) for x, y in zip(s0, state()))
    # a step whose emission would number ids past 2^32 - 1: refused before its deletions
    n = a.num_particles(f)
    ids = (np.arange(n, dtype=np.uint64) + (2 ** 32 - n - 2)).astype(np.uint32)
    a.set_ids(f, ids)
    a.delete_particles(f, np.arange(n) == 0)
    a.remove_source(P.sources[0][5])
    P.sources = []
    s = sheet(2, 0.5)
    a.add_source(f, s[0], None, 1)
    s1 = state()
    with pytest.raises(SphError):
        a.step(DT)
    assert all(same(x, y) for x, y in zip(s1, state()))


@pytest.mark.parametrize("marks", [False, True], ids=["no-marks", "marks"])
def test_id_overflow_on_the_device_path_changes_nothing(marks):
    """The world holds its truth on the device: the largest id comes from the classification (with host marks pending, from
    one without sinks, before the marks are applied).  The refused step leaves the particles, the last step's edits and the
    device scratch as they were (the world is not restaged: a staged world would read its densities as 0)."""
    sc = scene("xsph")
    sc["sources"] = []
    P = Pair(sc)
    a, f = P.a, P.fa[0]
    n = a.num_particles(f)
    a.set_ids(f, (np.arange(n, dtype=np.uint64) + (2 ** 32 - n - 2)).astype(np.uint32))
    a.step(DT)
    a.step(DT)
    a.add_source(f, sheet(2, 0.7)[0], None, 1)
    if marks:
        a.delete_particles(f, np.arange(a.num_particles(f)) == 0)

    def state():
        p, v = a.read_fluid(f)
        return dict(pos=p, vel=v, ids=a.read_ids(f), vc=a.debug(f, "velocity_change"), density=a.debug(f, "density"),
                    edits=np.array(a.step_edits(f)), n=np.array(a.num_particles(f)))

    s0 = state()
    assert np.abs(s0["density"]).max() > 0
    for _ in range(2):
        with pytest.raises(SphError):
            a.step(DT)
        s1 = state()
        assert [k for k in s0 if not same(s0[k], s1[k])] == []


def test_a_sink_removes_the_largest_id_in_a_firing_step():
    """The ids of a firing count from the largest id the fluid held at the start of the step, sunk particles included."""
    sc = scene("xsph")
    sc["sinks"], sc["sources"] = [], []
    P = Pair(sc)
    P.step()
    p, _ = P.a.read_fluid(P.fa[0])
    ids = P.a.read_ids(P.fa[0])
    top = p[np.argmax(ids)]
    P.add_sink(0, top, np.nextafter(top, F(np.inf)), 0)  # a box that holds exactly that particle
    s = sheet(2, 0.7)
    P.add_source(0, s[0], s[1], 5)
    assert P.step()[0] == (1, 4)
    now = P.a.read_ids(P.fa[0])
    assert ids.max() not in now and np.array_equal(np.sort(now)[-4:], ids.max() + 1 + np.arange(4))
    P.step()


def test_source_velocities_must_match_the_positions():
    w = LiquidWorld(particle_radius=R)
    f = w.add_fluid(sheet(2, 0.5)[0])
    with pytest.raises(ValueError):
        w.add_source(f, sheet(2, 0.5)[0], np.zeros((3, 3), F))


def test_slab_worlds_refuse_registration():
    w = LiquidWorld(particle_radius=R, slab_count=2)
    f = w.add_fluid(sheet(2, 0.5)[0])
    with pytest.raises(SphError):
        w.add_sink(f, (0, 0, 0), (1, 1, 1))
    with pytest.raises(SphError):
        w.add_source(f, sheet(2, 0.5)[0])


def test_domain_sink_bounds_the_grid():
    """A particle shot out of the tank at 1e4 m/s: with a domain sink around the tank every step runs and the grid stays
    within the domain's cells plus padding."""
    p, v = block(6, 6, 6, (0.1, 0.0, 0.1), 3, vy=0.0)
    v[0] = (1.0e4, 0.0, 0.0)
    w = LiquidWorld(particle_radius=R)
    f = w.add_fluid(p, velocities=v)
    w.add_boundary(TANK)
    lo, hi = np.array([-0.2, -1.0, -0.2], F), np.array([1.2, 2.0, 1.2], F)
    w.add_sink(f, lo, hi, outside=True)
    h = w.h
    cells = (np.floor(hi / F(h)) - np.floor(lo / F(h)) + 1).astype(int)
    for _ in range(20):
        w.step(DT)
        assert all(d <= c + 2 for d, c in zip(w.stats()["grid_dims"], cells))
    assert 0 not in w.read_ids(f)  # the fast particle left the domain and was removed


def test_a_sink_that_removes_nothing_costs_one_launch():
    p, v = block(6, 6, 6, (0.1, 0.0, 0.1), 3, vy=0.0)
    worlds = []
    for with_sink in (False, True):
        w = LiquidWorld(particle_radius=R)
        f = w.add_fluid(p, velocities=v)
        w.add_boundary(TANK)
        w.force_iterations(2, 3)
        if with_sink:
            w.add_sink(f, (-INF, -INF, -INF), (INF, -5.0, INF))
        worlds.append(w)
    for k in range(4):
        for w in worlds:
            w.step(DT)
        if k:
            assert worlds[1].stats()["kernel_launches"] == worlds[0].stats()["kernel_launches"] + 1
