"""sph_world_step_many (DESIGN.md section 13): K steps in one call, steps 2..K in a CUDA graph whose Jacobi loops end on the
device, against a twin world driven by K calls of step: state and per-step records bit-identical, the graph used where it
should be (on_device), its stops and fallbacks, the graph cache across host edits, and the refusals."""
import numpy as np
import pytest

from oracle import ref64_stages as S
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, SphError, StaticSampling, scenes
from salva_b200.liquid_world import Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

G = (0.0, -9.81, 0.0)
LIBS = pytest.mark.parametrize("lib", ["cubic", "poly6+spiky"])
PATHS = dict(
    quiet=(S.scene_block_forces, []),
    xsph=(S.scene_block, [scenes.xsph_viscosity(0.5, 0.0)]),
    artificial=(S.scene_block, [scenes.artificial_viscosity(0.2, 0.01, 0.0, 0.0, True)]),
    akinci_fused=(S.scene_block, [scenes.akinci2013_surface_tension(1.0, 0.0)]),
    akinci_adhesion=(S.scene_block, [scenes.akinci2013_surface_tension(1.0, 0.5)]),
    he2014=(S.scene_block, [scenes.he2014_surface_tension(1.0, 0.0)]),
    wcsph=(S.scene_block, [scenes.wcsph_surface_tension(1.0, 0.0)]),
    two_fluids=(S.scene_two_fluids, [scenes.xsph_viscosity(0.5, 0.0)]),
    sixteen=(S.scene_sixteen, []),
)


def _world(lib="cubic", solver="dfsph"):
    cls = DFSPHSolver if solver == "dfsph" else IISPHSolver
    s = cls(Poly6Kernel, SpikyKernel) if lib != "cubic" else cls()
    return LiquidWorld(s, particle_radius=S.R, smoothing_factor=2.0)


def _twins(scene, forces, lib="cubic", setup=None):
    out = []
    for _ in range(2):
        w = _world(lib)
        fh, bh = S.populate(w, scene(), forces)
        if setup:
            setup(w)
        out.append((w, fh, bh))
    return out


def _obs(w, fh, bh):
    o = {}
    for k, f in enumerate(fh):
        p, v = w.read_fluid(f)
        o["P%d" % k], o["V%d" % k] = p, v
        o["vc%d" % k] = w.debug(f, "velocity_change")
        o["id%d" % k] = w.read_ids(f)
    for k, b in enumerate(bh):
        o["bvol%d" % k], o["bf%d" % k] = w.read_boundary(b)
    return o


def _same(a, b, what):
    """Bit-identical, except the boundary forces: float atomics add them up in no fixed order, in two step() twins too."""
    assert a.keys() == b.keys()
    for k in a:
        if k.startswith("bf"):
            np.testing.assert_allclose(a[k], b[k], rtol=1e-5, atol=1e-6 * float(np.abs(b[k]).max() + 1.0), err_msg=what)
            continue
        assert np.array_equal(a[k], b[k]), "%s: %s differs (max |d| = %g)" % (what, k, float(np.abs(a[k] - b[k]).max()))


def _strip(recs):
    return [{k: v for k, v in r.items() if k != "on_device"} for r in recs]


def _drive(pair, K, dt=S.DT, gravity=G):
    """step_many(K) on the first world, K steps on the second; returns the first's records and the twin's."""
    (w1, f1, b1), (w2, f2, b2) = pair
    done = w1.step_many(dt, K, gravity=gravity)
    assert done == K
    rec1 = w1.step_records()
    rec2 = []
    _drive.twin_launches = 0
    for k in range(K):
        w2.step(dt, gravity)
        rec2 += w2.step_records()
        _drive.twin_launches += w2.stats()["kernel_launches"]
        if k == 0:
            _drive.first_launches = w2.stats()["kernel_launches"]
    _same(_obs(w1, f1, b1), _obs(w2, f2, b2), "step_many(%d)" % K)
    assert _strip(rec1) == _strip(rec2)
    return rec1


@LIBS
@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("K", [2, 3, 32])
def test_step_many_equals_steps(path, K, lib):
    scene, forces = PATHS[path]
    pair = _twins(scene, forces, lib)
    rec = _drive(pair, K)
    assert rec[0]["on_device"] == 0 and rec[1]["on_device"] == 1, [r["on_device"] for r in rec]
    st = pair[0][0].stats()
    assert st["n_substeps"] == K
    if all(r["on_device"] for r in rec[1:]):  # step 1's launches, the boundary sort on the envelope's grid, one graph launch
        assert st["kernel_launches"] <= _drive.first_launches + 16
    else:  # the block flew out of the envelope: some steps ran on the per-step path
        assert st["kernel_launches"] < _drive.twin_launches


def test_row_order(monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")
    for path in ("quiet", "xsph", "akinci_fused", "two_fluids"):
        scene, forces = PATHS[path]
        rec = _drive(_twins(scene, forces), 8)
        assert rec[1]["on_device"] == 1


def test_launches_do_not_grow_with_k():
    extra = []
    for K in (3, 4):
        pair = _twins(*PATHS["xsph"])
        _drive(pair, K)
        extra.append(pair[0][0].stats()["kernel_launches"] - _drive.first_launches)
    assert extra[0] == extra[1] and extra[0] <= 16, extra


# every way the loops can end, each with what the records of steps 2..K must show of it
LOOPS = dict(
    break0=(dict(min_div=0, min_press=0, loose=True), lambda r: r["n_divergence_eval"] == 1 and r["n_divergence_iter"] == 0
            and r["n_pressure_eval"] == 1 and r["n_pressure_iter"] == 0, any),
    break1=(dict(loose=True), lambda r: r["n_divergence_eval"] == 2 and r["n_divergence_iter"] == 1 and r["n_pressure_eval"] == 2
            and r["n_pressure_iter"] == 1, any),
    min0=(dict(min_div=0, min_press=0), lambda r: r["n_divergence_eval"] >= 1 and r["n_pressure_eval"] >= 1, all),
    min3=(dict(min_div=3, min_press=3), lambda r: r["n_divergence_eval"] >= 4 and r["n_pressure_eval"] >= 4, all),
    run_out2=(dict(max_div=2, max_press=2, tight=True), lambda r: r["n_divergence_iter"] == r["n_divergence_eval"] == 2
              and r["n_pressure_iter"] == r["n_pressure_eval"] == 2, all),
    run_out1=(dict(max_div=1, max_press=1), lambda r: r["n_divergence_eval"] == 1 and r["n_pressure_eval"] == 1, all),
    off_div=(dict(max_div=0, max_press=50), lambda r: r["n_divergence_eval"] == 0 and r["n_divergence_iter"] == 0
             and r["last_divergence_error"] == 0.0, all),
    off_press=(dict(max_div=50, max_press=0), lambda r: r["n_pressure_eval"] == 0 and r["n_pressure_iter"] == 0
               and r["last_density_error"] == 0.0, all),
    force00=(dict(force=(0, 0)), lambda r: (r["n_divergence_eval"], r["n_divergence_iter"], r["n_pressure_eval"], r["n_pressure_iter"]) == (1, 0, 1, 0), all),
    force12=(dict(force=(1, 2)), lambda r: (r["n_divergence_eval"], r["n_divergence_iter"], r["n_pressure_eval"], r["n_pressure_iter"]) == (2, 1, 3, 2), all),
    force31=(dict(force=(3, 1)), lambda r: (r["n_divergence_eval"], r["n_divergence_iter"], r["n_pressure_eval"], r["n_pressure_iter"]) == (4, 3, 2, 1), all),
)


@pytest.mark.parametrize("path", ["quiet", "xsph", "akinci_fused", "two_fluids"])
@pytest.mark.parametrize("loop", sorted(LOOPS))
def test_loop_ends(path, loop):
    scene, forces = PATHS[path]
    cfg, shows, quantifier = LOOPS[loop]

    def make():
        out = []
        for _ in range(2):
            s = DFSPHSolver()
            if "min_div" in cfg:
                s.min_divergence_iter, s.min_pressure_iter = cfg["min_div"], cfg["min_press"]
            if "max_div" in cfg:
                s.max_divergence_iter, s.max_pressure_iter = cfg["max_div"], cfg["max_press"]
            if cfg.get("loose"):
                s.max_divergence_error, s.max_density_error = 50.0, 0.5
            if cfg.get("tight"):
                s.max_divergence_error, s.max_density_error = 1e-9, 1e-9
            w = LiquidWorld(s, particle_radius=S.R, smoothing_factor=2.0)
            fh, bh = S.populate(w, scene(), forces)
            if "force" in cfg:
                w.force_iterations(*cfg["force"])
            out.append((w, fh, bh))
        return out

    rec = _drive(make(), 4)
    assert all(r["on_device"] == 1 for r in rec[1:]), [r["on_device"] for r in rec]
    assert quantifier(shows(r) for r in rec[1:]), rec


@pytest.mark.parametrize("scene", ["burst", "far"])
def test_envelope_exits(scene):
    sc = S.scene_burst if scene == "burst" else S.scene_far
    rec = _drive(_twins(sc, []), 12)
    if scene == "burst":
        assert any(r["on_device"] == 0 for r in rec[1:]), "the burst leaves the envelope"
    assert any(r["on_device"] == 1 for r in rec[1:])


def _cells(p, h):
    c = np.floor(p.astype(np.float32) / np.float32(h)).astype(np.int64)
    return c.min(0), c.max(0)


def test_lists_outgrow_headroom():
    """A block falling onto a finely sampled floor: its first step sees no boundary contact, so the boundary lists of the
    graph have 32 entries, and the floor brings ~90 per particle mid-call.  The graph stops after the search of that step,
    the step is redone on the per-step path, and the call goes on in a new graph; the fluid never leaves the envelope, so
    every per-step step after step 1 is such a redo."""
    g = np.arange(-0.3, 0.9, 0.025, dtype=np.float32)
    floor = np.stack(np.meshgrid(g, [0.0], g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    pts = scenes.block_lattice(6, 6, 6, S.R, origin=(0.0, 0.3, 0.0)).astype(np.float32)
    vel = np.tile(np.array([[0.0, -3.0, 0.0]], np.float32), (len(pts), 1))
    sc = lambda: dict(fluids=[dict(positions=pts, velocities=vel, density0=1000.0)], boundaries=[dict(positions=floor)])
    pair = _twins(sc, [])
    (w1, f1, b1), (w2, f2, b2) = pair
    K = 24
    assert w1.step_many(S.DT, K, gravity=(0.0, 0.0, 0.0)) == K
    rec1 = w1.step_records()
    rec2 = []
    h = w2.h
    for k in range(K):
        w2.step(S.DT, (0.0, 0.0, 0.0))
        rec2 += w2.step_records()
        lo, hi = _cells(w2.read_fluid(f2[0])[0], h)
        if k == 0:
            blo, bhi = _cells(floor, h)
            env_lo, env_hi = np.minimum(lo, blo) - 4, np.maximum(hi, bhi) + 4
        else:
            assert (lo >= env_lo).all() and (hi <= env_hi).all(), "the fluid left the envelope at step %d" % (k + 1)
    _same(_obs(w1, f1, b1), _obs(w2, f2, b2), "lists outgrow the headroom")
    assert _strip(rec1) == _strip(rec2)
    redo = [k for k in range(1, K) if rec1[k]["on_device"] == 0]
    assert redo, [r["on_device"] for r in rec1]
    assert any(k + 1 < K and rec1[k + 1]["on_device"] == 1 for k in redo), [r["on_device"] for r in rec1]


def _zero_mass():
    r = 0.05
    pts = scenes.jitter(scenes.block_lattice(6, 6, 6, r * 0.8), r, 3)
    tank = scenes.open_tank((-r, -r, -r), (12 * r, 0.8, 12 * r), r)
    return dict(fluids=[dict(positions=pts, density0=0.0)], boundaries=[dict(positions=tank)])


def test_zero_mass_fails_like_step():
    w1, w2 = LiquidWorld(particle_radius=0.05), LiquidWorld(particle_radius=0.05)
    scenes.populate(w1, _zero_mass())
    scenes.populate(w2, _zero_mass())
    with pytest.raises(SphError, match="zero density") as e1:
        w1.step_many(S.DT, 5)
    with pytest.raises(SphError, match="zero density") as e2:
        w2.step(S.DT)
    assert e1.value.status == e2.value.status
    assert len(w1.step_records()) == 1


def test_non_finite_velocity_fails_like_step():
    pair = _twins(*PATHS["quiet"])
    for w, fh, _ in pair:
        p, v = w.read_fluid(fh[0])
        v[3] = np.inf
        w.write_fluid(fh[0], velocities=v)
    errs = []
    for k, (w, fh, _) in enumerate(pair):
        done = 0
        try:
            if k == 0:
                w.step_many(S.DT, 5)
            else:
                for _ in range(5):
                    w.step(S.DT)
                    done += 1
        except SphError as e:
            errs.append((e.status, e.steps_done if k == 0 else done))
    assert len(errs) == 2 and errs[0] == errs[1], errs


def test_cache_across_host_edits():
    pair = _twins(*PATHS["xsph"])
    _drive(pair, 5)
    for w, fh, _ in pair:
        p, v = w.read_fluid(fh[0])
        w.write_fluid(fh[0], velocities=v * 0.5)
    _drive(pair, 5)
    for w, fh, _ in pair:
        w.append_particles(fh[0], np.array([[0.3, 0.5, 0.3]], np.float32))
    _drive(pair, 5)
    for w, fh, _ in pair:
        m = np.zeros(w.num_particles(fh[0]), np.uint8)
        m[::7] = 1
        w.delete_particles(fh[0], m)
    _drive(pair, 5)
    _drive(pair, 5, dt=S.DT * 0.5)
    _drive(pair, 5, gravity=(0.0, -5.0, 1.0))
    for w, fh, _ in pair:
        w.force_iterations(2, 2)
    _drive(pair, 4)
    for w, fh, _ in pair:
        w.force_iterations(-1, -1)
    blob = pair[0][0].snapshot()
    _drive(pair, 5)
    for w, fh, _ in pair:
        w.restore(blob)
    _drive(pair, 5)


def test_remove_fluid_between_calls():
    pair = _twins(*PATHS["two_fluids"])
    _drive(pair, 4)
    for w, fh, _ in pair:
        w.remove_fluid(fh[1])
    (w1, f1, b1), (w2, f2, b2) = pair
    w1.step_many(S.DT, 4)
    for _ in range(4):
        w2.step(S.DT)
    _same(_obs(w1, f1[:1], b1), _obs(w2, f2[:1], b2), "after remove_fluid")


def test_snapshot_after_step_many_continues():
    (w1, f1, b1), = _twins(*PATHS["akinci_fused"])[:1]
    w1.step_many(S.DT, 6)
    blob = w1.snapshot()
    w1.step_many(S.DT, 4)
    a = _obs(w1, f1, b1)
    w1.restore(blob)
    for _ in range(4):
        w1.step(S.DT)
    _same(a, _obs(w1, f1, b1), "snapshot continuation")


def _refused(w, fh, bh):
    before = _obs(w, fh, bh)
    with pytest.raises(SphError) as e:
        w.step_many(S.DT, 3)
    assert "INVALID" in str(e.value)
    _same(before, _obs(w, fh, bh), "refusal")
    w.step(S.DT)


def test_refusals_change_nothing():
    w = _world(solver="iisph")
    fh, bh = S.populate(w, S.scene_block(), [])
    _refused(w, fh, bh)
    for forces in ([scenes.becker2009_elasticity(2.0e5, 0.3)], [scenes.dfsph_viscosity(0.1, 0.1)]):
        w = _world()
        fh, bh = S.populate(w, S.scene_block(), forces)
        _refused(w, fh, bh)
    w = _world()
    fh, bh = S.populate(w, S.scene_block(), [])
    w.push_host_force(fh[0], lambda *a: None)
    _refused(w, fh, bh)
    w = _world()
    fh, bh = S.populate(w, S.scene_block(), [])
    w.set_substepping(0.4)
    _refused(w, fh, bh)
    w = _world()
    fh, bh = S.populate(w, S.scene_block(), [])
    box = scenes.cuboid_surface((0.1, 0.08, 0.1), S.R).astype(np.float32)
    w.register_coupling(w.add_boundary(np.zeros((0, 3), np.float32)), StaticSampling(box))
    _refused(w, fh, bh)
    slab = LiquidWorld(particle_radius=S.R, slab_rank=0, slab_count=2)
    with pytest.raises(SphError) as e:
        slab.step_many(S.DT, 3)
    assert e.value.status == 1
    w = _world()
    fh, bh = S.populate(w, S.scene_block(), [])
    before = _obs(w, fh, bh)
    assert w.step_many(S.DT, 0) == 0
    _same(before, _obs(w, fh, bh), "n_steps = 0")


def test_c1_200_steps():
    out = []
    for k in range(2):
        w = LiquidWorld(particle_radius=0.05, smoothing_factor=2.0)
        fh, bh = scenes.populate(w, scenes.scene_c1())
        if k == 0:
            assert w.step_many(1.0 / 200.0, 200) == 200
            assert sum(r["on_device"] for r in w.step_records()) >= 150
        else:
            for _ in range(200):
                w.step(1.0 / 200.0)
        out.append(np.concatenate(w.read_fluid(fh[0])))
    assert np.array_equal(out[0], out[1])
