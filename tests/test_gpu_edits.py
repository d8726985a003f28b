"""Host edits of a running world, checked against oracle/edit_model.py: append, delete, write (host-staged and device path),
remove_fluid, add_fluid into a reused slot, replace_particles, set_ids, snapshot / restore.

Edits are permutations, filters and splices of what a particle carries (position, velocity, velocity_change, IISPH pressure,
volume, id, deletion mark, its fluid's offset), so after every operation the world must agree with the model BIT FOR BIT:
(a) seeded edit programs, every read-back compared after every operation;
(b) at several points of each program the edited world must continue exactly like a fresh world restored from its snapshot
    (and, one default-volume DFSPH fluid, like one rebuilt through replace_particles in a shuffled order);
(c) the density pass of the step after the program against oracle/ref64.py on the model's volumes and fluid assignment,
    which no read-back exposes;
(d) the programs the CPU oracle can follow, against it;
(e) edges: buffer growth, the cached grid bounds, an emptied world, removal and restore with marks pending, scratch validity,
    Becker-2009 with a delete and an append that cancel, boundary edits interleaved with fluid edits under colliders.
tests/test_edit_model.py runs the same programs without a GPU against mutants of the model.
"""
import os

import numpy as np
import pytest

from oracle import edit_model as em
from oracle.oracle import OracleWorld
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, scenes
from salva_b200.liquid_world import Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

F = np.float32
R = 0.05
DT = 0.004
NX, NZ = 10, 8
SEEDS = (1, 2, 3)
SCENE_SEED = dict(dfsph1=1000, dfsph3=3000, iisph2=2000)  # the programs of two scenes do not share their order


def _block(ny, y0, seed):
    rng = np.random.default_rng(seed)
    p = scenes.jitter(scenes.block_lattice(NX, ny, NZ, R * 0.93, origin=(0.0, y0, 0.0)), R, seed, amplitude=0.3)
    return p, rng.normal(0, 0.2, p.shape).astype(F)


def make_scene(name):
    """dfsph1: one fluid with XSPH (velocity_changes and the fused paths matter); dfsph3: three fluids, the middle one with
    per-particle volumes, the third in an interaction group the second does not see, artificial viscosity; iisph2: two fluids
    under IISPH (pressures are carried)."""
    s = 2 * R * 0.93
    if name == "dfsph1":
        p, v = _block(9, 0.0, 3)
        fluids = [dict(positions=p, velocities=v, density0=1000.0, forces=[scenes.xsph_viscosity(0.5, 0.2)])]
        top, solver = 9 * s, scenes.DFSPH
    elif name == "dfsph3":
        fluids = []
        for k, rho in enumerate((1000.0, 900.0, 800.0)):
            p, v = _block(4, 4 * k * s, 5 + k)
            fluids.append(dict(positions=p, velocities=v, density0=rho, forces=[scenes.artificial_viscosity(1.0, 0.0)]))
        fluids[1]["volumes"] = (em.default_volume(R) * np.random.default_rng(9).uniform(0.9, 1.1, len(p))).astype(F)
        fluids[1]["filter"] = 0xFFFFFFFF ^ 2
        fluids[2]["memberships"] = 2
        top, solver = 12 * s, scenes.DFSPH
    else:
        fluids = []
        for k, rho in enumerate((1000.0, 800.0)):
            p, v = _block(5, 5 * k * s, 11 + k)
            fluids.append(dict(positions=p, velocities=v, density0=rho, forces=[scenes.artificial_viscosity(1.0, 0.0)]))
        top, solver = 10 * s, scenes.IISPH
    tank = scenes.open_tank((-R, -R, -R), (NX * 2 * R + R, 1.2, NZ * 2 * R + R), R)
    return dict(name=name, solver=solver, fluids=fluids, boundaries=[dict(positions=tank)], top=top + 0.15)


def populate(world, model, scene):
    """The scene into a world (None: the model alone) and its model; the two must hand out the same handles."""
    for f in scene["fluids"]:
        kw = dict(density0=f["density0"], velocities=f.get("velocities"), volumes=f.get("volumes"),
                  memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF))
        h = model.add_fluid(f["positions"], **kw)
        for force in f["forces"]:
            model.push_force(h, *force)
        if world is not None:
            assert world.add_fluid(f["positions"], **kw) == h
            for force in f["forces"]:
                world.push_force(h, *force)
    return [world.add_boundary(b["positions"]) for b in scene["boundaries"]] if world is not None else []


def programs(name, host_only=True, seeds=SEEDS, n_fill=10):
    """(scene, [operations, ...]): the programs of one scene, the same on every machine."""
    scene = make_scene(name)
    model = em.EditModel(R)
    populate(None, model, scene)
    per_volume = model.handles()[1] if name == "dfsph3" else None
    out = []
    for seed in seeds:
        layers = em.Layers(R, NX, NZ, scene["top"])
        out.append(em.make_program(SCENE_SEED[name] + seed, model, layers, DT, n_fill=n_fill, host_only=host_only, per_volume=per_volume))
    return scene, out


# ---- worlds ----------------------------------------------------------------------------------------------------------------
CONFIGS = {"cubic": dict(), "row": dict(row=True), "generic": dict(generic=True)}


def make_world(scene, row=False, generic=False):
    """cubic: the cubic-spline library in h-cell order; row: the same in row order (read when the world is created);
    generic: the generic-kernel library (Poly6 density, Spiky gradient)."""
    S = IISPHSolver if scene["solver"] == scenes.IISPH else DFSPHSolver
    solver = S(Poly6Kernel, SpikyKernel) if generic else S()
    old = os.environ.get("SALVA_B200_XYSUB")
    os.environ["SALVA_B200_XYSUB"] = "2" if row else "1"
    try:
        return LiquidWorld(solver, particle_radius=R, smoothing_factor=2.0)
    finally:
        if old is None:
            del os.environ["SALVA_B200_XYSUB"]
        else:
            os.environ["SALVA_B200_XYSUB"] = old


def world_like(model, scene, cfg):
    """A fresh world with the model's slot table: the same live and dead slots, rest densities, groups and forces, one
    placeholder particle per fluid (a restore or replace_particles brings the real ones).  Handles are the slot numbers."""
    w = make_world(scene, **cfg)
    for s in model.slots:
        h = w.add_fluid(s.pos[:1] if s.n else np.zeros((1, 3), F), density0=float(s.density0), memberships=s.memberships, filter=s.filter)
        for force in s.forces:
            w.push_force(h, *force)
    for k, s in enumerate(model.slots):
        if not s.alive:
            w.remove_fluid(k)
    for b in scene["boundaries"]:
        w.add_boundary(b["positions"])
    return w


def by_id(world, handle, pressures):
    got = em.read_world(world, handle, pressures)
    ids = got.pop("id")
    assert len(np.unique(ids)) == len(ids), "fluid %#x holds %d particles under %d ids" % (handle, len(ids), len(np.unique(ids)))
    o = np.argsort(ids)
    return ids[o], {k: v[o] for k, v in got.items()}


def assert_same_continuation(a, others, model, pressures, steps=4):
    """Step `a` and every world of `others` (world, handle of slot k) and compare, particle by particle matched by id."""
    for _ in range(steps):
        model.begin_step()
        a.step(DT)
        for w, _ in others:
            w.step(DT)
    for k, s in enumerate(model.slots):
        if not s.alive:
            continue
        ha = k | s.gen << 16
        ia, sa = by_id(a, ha, pressures)
        for w, handle_of in others:
            ib, sb = by_id(w, handle_of(k), pressures)
            assert np.array_equal(ia, ib)
            for name in sa:
                d = em._first_diff(name, ha, sb[name], sa[name])
                if d:
                    first = int(np.nonzero((sa[name] != sb[name]).reshape(len(ia), -1).any(axis=1))[0][0])
                    raise AssertionError("a rebuilt world diverged from the edited one after %d steps (rebuilt, edited): %s; its id is %d"
                                         % (steps, d, ia[first]))
    em.refresh_from(a, model, pressures)


def continuation_check(a, model, scene, cfg, pressures, replace_route):
    """(b), called after a step of DT: a fresh world restored from a's snapshot, and optionally one rebuilt with
    replace_particles in a shuffled order after one step of DT (the lagging timestep is the one thing replace_particles
    does not bring), continue bit-identically to a."""
    blob = a.snapshot()
    model.snapshot()
    b = world_like(model, scene, cfg)
    b.restore(blob)
    others = [(b, lambda k: k)]
    if replace_route:
        c = world_like(model, scene, cfg)
        c.step(DT)
        s = model.slots[0]
        perm = np.random.default_rng(s.n).permutation(s.n)
        c.replace_particles(0, s.pos[perm], s.vel[perm], s.vc[perm], s.id[perm])
        others.append((c, lambda k: k))
    assert_same_continuation(a, others, model, pressures)
    for w, _ in others:
        w.close()


def mass_step(a, model, scene, cfg, bh, pressures):
    """(c): one step whose density pass is checked against ref64 on the model's volumes, rest densities and fluid assignment."""
    model.begin_step()
    ps = em.passes_of(model, a.h, scene["boundaries"], **(dict(kw=1, kg=2) if cfg.get("generic") else {}))
    a.step(DT)
    live = [h for h in model.handles() if model.slot(h).n]
    cat = lambda what: np.concatenate([a.debug(h, what) for h in live])  # noqa: E731
    bvol = np.concatenate([a.read_boundary(b)[0] for b in bh])
    bad = em.mass_mismatches(ps, cat("density"), cat("num_fluid_contacts"), cat("num_boundary_contacts"), bvol,
                             alpha=None if pressures else cat("alpha"))
    assert not bad, "\n".join(bad)
    bad = em.mismatches(a, model, pressures, after_step=True)
    assert not bad, "\n".join(bad)
    em.refresh_from(a, model, pressures)


def run_program(scene, ops, cfg, totals):
    pressures = scene["solver"] == scenes.IISPH
    a, model = make_world(scene, **cfg), em.EditModel(R)
    bh = populate(a, model, scene)
    assert em.has_collision_pattern(ops, model), "the program must hold delete -> step -> append with a surviving id above the count"
    assert not em.mismatches(a, model, pressures)
    totals["particles"] = max(totals["particles"], sum(model.slot(h).n for h in model.handles()))
    state = {}
    for k, op in enumerate(ops):
        if op[0] == "rebuild":
            mass_step(a, model, scene, cfg, bh, pressures)
            continuation_check(a, model, scene, cfg, pressures, replace_route=scene["name"] == "dfsph1")
            totals["rebuilds"] += 1
            continue
        bad = em.apply_op(a, model, op, state, pressures)
        assert not bad, "after operation %d %s:\n" % (k, op[0]) + "\n".join(bad)
        totals["ops"] += 1
    mass_step(a, model, scene, cfg, bh, pressures)
    a.close()


@pytest.mark.parametrize("name,config", [("dfsph1", "cubic"), ("dfsph1", "row"), ("dfsph3", "cubic"), ("dfsph3", "generic"),
                                         ("iisph2", "cubic"), ("iisph2", "row")])
def test_edit_programs_agree_with_the_model_bit_for_bit(name, config):
    scene, progs = programs(name)
    totals = dict(ops=0, rebuilds=0, particles=0)
    for ops in progs:
        run_program(scene, ops, CONFIGS[config], totals)
    print("%s/%s: %d programs, %d operations, %d continuation checks, up to %d particles" % (name, config, len(progs), totals["ops"],
                                                                                          totals["rebuilds"], totals["particles"]))


def test_append_after_delete_and_step_gives_ids_no_survivor_holds():
    """100 particles, delete 30, step, append 20: ids numbered from the shrunken count (70..89) would repeat the ids of
    survivors, and the in-cell order (fluid, id) would then depend on the previous order: a twin that is left alone and a
    world restored from a snapshot would drift apart in the last bits."""
    scene = make_scene("dfsph1")
    worlds = []
    for _ in range(2):
        w, m = make_world(scene), em.EditModel(R)
        populate(w, m, scene)
        h = m.handles()[0]
        n = m.slot(h).n
        mask = np.zeros(n, bool)
        mask[np.random.default_rng(0).choice(n - 200, 230, replace=False)] = True   # the last 200 ids survive
        extra = em.Layers(R, NX, NZ, scene["top"]).take(60)
        for op in (("step", DT), ("delete", h, mask), ("step", DT), ("append", h, extra, None), ("step", DT), ("step", DT), ("step", DT)):
            bad = em.apply_op(w, m, op, {})
            assert not bad, "\n".join(bad)
        worlds.append((w, m))
    (a, ma), (twin, _) = worlds
    ids = a.read_ids(h)
    assert len(np.unique(ids)) == len(ids) == n - 230 + 60 and ids[-60:].min() == n
    b = world_like(ma, scene, {})
    b.restore(twin.snapshot())   # a itself is not disturbed: it keeps the order its steps left on the device
    assert_same_continuation(a, [(b, lambda k: k)], ma, False)


# ---- (d) the oracle ------------------------------------------------------------------------------------------------------------
def _oracle_apply(cpu, op):
    kind = op[0]
    if kind == "step":
        cpu.step(op[1])
    elif kind == "append":
        cpu.append_particles(op[1], op[2], op[3])
    elif kind == "delete":
        cpu.delete_particles(op[1], op[2])
    elif kind == "write":
        p, v = cpu.read_fluid(op[1])
        cpu.write_fluid(op[1], None if op[2] is None else (p + op[2]).astype(F), None if op[3] is None else (v + op[3]).astype(F))


@pytest.mark.parametrize("name,config", [("dfsph1", "cubic"), ("dfsph3", "generic"), ("iisph2", "row")])
def test_edit_programs_follow_the_oracle(name, config):
    """Counts after every operation, contact counts while the two worlds still hold bit-identical positions (the first
    step), and max |dx| <= 1e-3 h at the end of every program the oracle has the operations for."""
    scene, progs = programs(name, host_only=False, n_fill=3)
    cfg = CONFIGS[config]
    for ops in progs:
        gpu, model = make_world(scene, **cfg), em.EditModel(R)
        populate(gpu, model, scene)
        kd, kg = (1, 2) if cfg.get("generic") else (0, 0)
        cpu = OracleWorld(R, 2.0, solver=scene["solver"], kernel_density=kd, kernel_gradient=kg)
        for f in scene["fluids"]:
            h = cpu.add_fluid(f["positions"], density0=f["density0"], velocities=f.get("velocities"), volumes=f.get("volumes"),
                              memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF))
            for force in f["forces"]:
                cpu.push_force(h, *force)
        for b in scene["boundaries"]:
            cpu.add_boundary(b["positions"])
        for w in (gpu, cpu):
            w.force_iterations(1, 2)
        stepped, state = False, {}
        for op in ops:
            if op[0] == "rebuild":
                continue
            first = op[0] == "step" and not stepped
            bad = em.apply_op(gpu, model, op, state, scene["solver"] == scenes.IISPH)
            assert not bad, "\n".join(bad)
            _oracle_apply(cpu, op)
            for h in model.handles():
                assert gpu.num_particles(h) == cpu.num_particles(h)
                if first and model.slot(h).n:
                    for what in ("num_fluid_contacts", "num_boundary_contacts"):
                        assert np.array_equal(gpu.debug(h, what), cpu.debug(h, what))
            stepped |= op[0] == "step"
        for h in model.handles():
            if model.slot(h).n:
                assert np.abs(gpu.read_fluid(h)[0] - cpu.read_fluid(h)[0]).max() <= 1e-3 * float(gpu.h)
        gpu.close()


# ---- (e) edges -----------------------------------------------------------------------------------------------------------------
def _small(n):
    """n particles of a 10 x ? x 8 block in the tank, one DFSPH fluid with XSPH"""
    scene = make_scene("dfsph1")
    f = scene["fluids"][0]
    f["positions"], f["velocities"] = f["positions"][:n].copy(), f["velocities"][:n].copy()
    return scene


def test_growth_past_a_multiple_of_32_and_past_the_allocated_buffers():
    scene = _small(250)
    a, model = make_world(scene), em.EditModel(R)
    populate(a, model, scene)
    h = model.handles()[0]
    layers = em.Layers(R, NX, NZ, scene["top"])
    ops = [("step", DT), ("append", h, layers.take(5), None), ("step", DT), ("append", h, layers.take(2), None), ("step", DT)]   # 255 -> 257
    big = np.concatenate([layers.take(80) for _ in range(10)])                                                                 # several times N
    ops += [("append", h, big, np.zeros_like(big)), ("step", DT), ("step", DT)]
    state = {}
    for op in ops:
        bad = em.apply_op(a, model, op, state)
        assert not bad, "\n".join(bad)
    assert a.num_particles(h) == 1057 and a.stats()["n_fluid_particles"] == 1057
    continuation_check(a, model, scene, {}, False, replace_route=True)


def test_edits_outside_the_cached_grid_bounds():
    """An append far outside the bounds the last step cached, and a write that moves the whole block outside them: the next
    step's grid covers the new extent and the contact counts are the oracle's."""
    scene = _small(400)
    gpu, model = make_world(scene), em.EditModel(R)
    populate(gpu, model, scene)
    cpu = OracleWorld(R, 2.0)
    fc, _ = scenes.populate(cpu, scene)
    h = model.handles()[0]
    far = (em.Layers(R, 3, 3, 0.3).take(9) + np.array([7.3, 0.0, -5.1], F)).astype(F)
    for w, f in ((gpu, h), (cpu, fc[0])):
        w.step(DT)
        w.step(DT)
    dims0 = gpu.stats()["grid_dims"]
    for w, f in ((gpu, h), (cpu, fc[0])):
        w.append_particles(f, far)
        w.step(DT)
    dims1 = gpu.stats()["grid_dims"]
    hh = float(gpu.h)
    assert dims1[0] >= dims0[0] + int(6.0 / hh) and dims1[2] >= dims0[2] + int(4.0 / hh)
    p = gpu.read_fluid(h)[0]
    moved = (p + np.array([-9.0, 2.0, 0.0], F)).astype(F)   # the device path of write, right after a step
    for w, f in ((gpu, h), (cpu, fc[0])):
        w.write_fluid(f, positions=moved, velocities=np.zeros_like(moved))
        w.step(DT)
    dims2 = gpu.stats()["grid_dims"]
    assert dims2[0] >= int(9.0 / hh) and dims2[1] >= int(2.0 / hh)
    for what in ("num_fluid_contacts", "num_boundary_contacts"):
        assert np.array_equal(gpu.debug(h, what), cpu.debug(fc[0], what))
    assert np.array_equal(gpu.debug(h, "num_boundary_contacts"), np.zeros(len(moved), F))


def test_every_particle_deleted_then_stepped_then_appended_again():
    scene = _small(300)
    a, model = make_world(scene), em.EditModel(R)
    populate(a, model, scene)
    h = model.handles()[0]
    again = em.Layers(R, NX, NZ, scene["top"]).take(70)
    state = {}
    for op in (("step", DT), ("delete", h, np.ones(300, bool)), ("step", DT), ("step", DT), ("append", h, again, None), ("step", DT),
               ("step", DT)):
        bad = em.apply_op(a, model, op, state)
        assert not bad, "\n".join(bad)
    assert a.num_particles(h) == 70 and np.array_equal(a.read_ids(h), np.arange(70, dtype=np.uint32))
    assert np.isfinite(a.read_fluid(h)[0]).all()
    continuation_check(a, model, scene, {}, False, replace_route=True)


def test_append_is_refused_when_the_new_ids_would_not_fit_32_bits():
    scene = _small(100)
    w, model = make_world(scene), em.EditModel(R)
    populate(w, model, scene)
    h = model.handles()[0]
    ids = np.arange(100, dtype=np.uint32)
    ids[17] = 0xFFFFFFFE
    w.set_ids(h, ids)
    new = em.Layers(R, NX, NZ, scene["top"]).take(2)
    with pytest.raises(Exception):
        w.append_particles(h, new)            # 0xFFFFFFFF and one past it
    assert w.num_particles(h) == 100 and np.array_equal(w.read_ids(h), ids)
    w.append_particles(h, new[:1])
    assert w.read_ids(h)[-1] == 0xFFFFFFFF
    w.step(DT)
    assert w.num_particles(h) == 101


def test_removal_and_restore_with_marks_pending():
    """A fluid removed while particles of it are marked; a restore into a world whose fluid has marks pending and another
    count: neither the marks nor the count may survive."""
    scene = make_scene("iisph2")
    a, model = make_world(scene), em.EditModel(R)
    populate(a, model, scene)
    h0, h1 = model.handles()
    rng = np.random.default_rng(4)
    state = {}
    ops = [("step", DT), ("step", DT), ("snapshot",), ("step", DT),
           ("append", h1, em.Layers(R, NX, NZ, scene["top"]).take(33), None),
           ("delete", h1, rng.random(model.slot(h1).n + 33) < 0.2), ("delete", h0, rng.random(model.slot(h0).n) < 0.2),
           ("restore",), ("step", DT), ("delete", h0, rng.random(model.slot(h0).n) < 0.3), ("remove", h0), ("step", DT), ("step", DT)]
    for op in ops:
        bad = em.apply_op(a, model, op, state, pressures=True)
        assert not bad, "%s:\n" % op[0] + "\n".join(bad)
    assert a.num_particles(h1) == len(scene["fluids"][1]["positions"])
    continuation_check(a, model, scene, {}, True, replace_route=False)


def _block_scene(n, seed, forces):
    """an n^3 block at rest spacing, jittered and stirred, in the tank"""
    rng = np.random.default_rng(seed)
    p = scenes.jitter(scenes.block_lattice(n, n, n, R), R, seed, amplitude=0.3)
    tank = scenes.open_tank((-R, -R, -R), (n * 2 * R + R, 1.2, n * 2 * R + R), R)
    return dict(name="block", solver=scenes.DFSPH, boundaries=[dict(positions=tank)], top=n * 2 * R + 0.15,
                fluids=[dict(positions=p, velocities=rng.normal(0, 0.2, p.shape).astype(F), density0=1000.0, forces=list(forces))])


@pytest.mark.parametrize("force,selectors", [(scenes.he2014_surface_tension(1.0, 0.5), (12, 13)), (scenes.dfsph_viscosity(0.3, 1, 1, 0.01), (14, 15)),
                                             (scenes.becker2009_elasticity(1.0e5, 0.3, True), (16, 17, 18, 19))],
                         ids=["he2014", "viscosity", "becker"])
def test_plugin_scratch_follows_the_particle_set(force, selectors):
    """include/sph.h: the selectors of a plugin's scratch are refused unless its force was solved since particles were last
    added or deleted; after a write they hold the last solve's values.  DFSPHViscosity runs one iteration: the reference's loop
    amplifies its error on such a scene (tests/test_gpu_parity.py::test_dfsph_viscosity_row_a16), here and in the oracle alike."""
    scene = _block_scene(8, 21, [force])
    w, model = make_world(scene), em.EditModel(R)
    populate(w, model, scene)
    h = model.handles()[0]
    n = w.num_particles(h)

    def refused():
        for s in selectors:
            with pytest.raises(Exception):
                w.debug(h, s)

    def accepted(count):
        for s in selectors:
            got = w.debug(h, s)
            assert len(got) == count and np.isfinite(got).all(), "selector %d" % s

    refused()                                           # never solved
    w.step(DT)
    kept = {s: w.debug(h, s) for s in selectors}
    p, v = w.read_fluid(h)
    w.write_fluid(h, positions=p, velocities=v)
    for s in selectors:
        assert np.array_equal(w.debug(h, s), kept[s]), "selector %d after a write" % s
    w.append_particles(h, em.Layers(R, 8, 8, scene["top"]).take(5))
    refused()                                           # added
    w.step(DT)
    accepted(n + 5)                                     # solved again
    mask = np.zeros(n + 5, bool)
    mask[::7] = True
    w.delete_particles(h, mask)
    w.snapshot()                                        # applies the marks without solving anything
    assert w.num_particles(h) == n + 5 - int(mask.sum())
    refused()                                           # deleted
    w.step(DT)
    accepted(n + 5 - int(mask.sum()))


def test_becker_keeps_its_rest_pose_when_a_delete_and_an_append_cancel():
    """Becker-2009 recaptures its rest pose when the particle count changes (becker2009_elasticity.rs:87).  A delete and an
    append of equal size in one interval leave the count as it was, so the reference does not recapture, and neither may the
    engine: the rest volumes stay, and the trajectory stays the oracle's."""
    scene = _block_scene(8, 9, [scenes.becker2009_elasticity(1.0e5, 0.3, True)])
    gpu, model = make_world(scene), em.EditModel(R)
    populate(gpu, model, scene)
    h = model.handles()[0]
    cpu = OracleWorld(R, 2.0)
    (o,), _ = scenes.populate(cpu, scene)
    for w in (gpu, cpu):
        w.force_iterations(1, 2)
        w.step(DT)
        w.step(DT)
    rest_gpu, rest_cpu = gpu.debug(h, "el_volume0"), cpu.debug(o, "el_volume0")
    assert np.abs(rest_gpu - rest_cpu).max() <= 1e-5 * np.abs(rest_cpu).max()
    p, v = gpu.read_fluid(h)
    n, k = len(p), 20
    mask = np.zeros(n, bool)
    mask[-k:] = True                                     # the new particles take the indices of the ones that go
    new = (p[-k:] + np.array([0.0, 0.2 * R, 0.0], F)).astype(F)
    for w, f in ((gpu, h), (cpu, o)):
        w.delete_particles(f, mask)
        w.append_particles(f, new, v[-k:])
        w.step(DT)
    assert gpu.num_particles(h) == cpu.num_particles(o) == n
    assert np.array_equal(gpu.debug(h, "el_volume0"), rest_gpu), "the engine recaptured the rest pose"
    assert np.array_equal(cpu.debug(o, "el_volume0"), rest_cpu)
    for w in (gpu, cpu):
        w.step(DT)
        w.step(DT)
    assert np.abs(gpu.read_fluid(h)[0] - cpu.read_fluid(o)[0]).max() <= 1e-3 * float(gpu.h)
    # one particle more: the count changes and the rest pose is captured again, from the deformed state
    gpu.append_particles(h, em.Layers(R, 8, 8, scene["top"]).take(1))
    gpu.step(DT)
    assert not np.array_equal(gpu.debug(h, "el_volume0")[:n], rest_gpu)


def test_boundary_edits_interleaved_with_fluid_edits_match_a_world_built_in_the_final_configuration():
    """Boundary 2 belongs to a StaticSampling collider and boundary 3 to a contact-sampling one, so the engine keeps the
    boundaries on the device.  Boundary 0 is removed and a larger one added into its slot, boundary 1 gets another particle
    set, the fluid is appended to and deleted from in between.  The world then steps bit for bit like one built directly
    in the final configuration, and every boundary reads back its own particles."""
    from salva_b200 import BODY_FIXED, StaticSampling
    from salva_b200.liquid_world import Ball, DynamicContactSampling
    base = _small(400)
    tank = base["boundaries"][0]["positions"]
    lid = scenes._face(1, 1.1, (0.0, 0.0, 0.0), (0.5, 0.0, 0.4), 2 * R)
    lid2 = scenes._face(1, 1.0, (0.0, 0.0, 0.0), (0.9, 0.0, 0.7), 2 * R)
    bigger = np.concatenate([tank, scenes._face(1, 1.25, (0.0, 0.0, 0.0), (0.9, 0.0, 0.7), 2 * R)])
    assert len(lid2) != len(lid) and len(bigger) > len(tank)
    box = scenes.cuboid_surface((0.1, 0.05, 0.1), R)
    box_at = (np.array([0.8, 0.3, 0.4], F), np.array([0.78, 0.34, 0.42], F))
    ball_at = np.array([0.3, 0.92, 0.4], F)

    def build(b0, b1):
        scene = dict(base, boundaries=[dict(positions=b0), dict(positions=b1)])
        w, model = make_world(scene), em.EditModel(R)
        bh = populate(w, model, scene)
        bh += [w.add_boundary(np.zeros((0, 3), F)), w.add_boundary(np.zeros((0, 3), F))]
        cs = w.register_coupling(bh[2], StaticSampling(box))
        cc = w.register_coupling(bh[3], DynamicContactSampling(Ball(0.1)))
        w.set_collider_state(cs, translation=box_at[0], body=BODY_FIXED)
        w.set_collider_state(cc, translation=ball_at)
        return w, model, bh, cs

    x, model, bx, cs_x = build(tank, lid)
    h = model.handles()[0]
    state = {}

    def edit(op):
        bad = em.apply_op(x, model, op, state)
        assert not bad, "\n".join(bad)

    edit(("step", DT))
    edit(("step", DT))
    assert len(x.read_boundary_particles(bx[3])[0]) > 0, "the ball must sample the fluid"
    x.remove_boundary(bx[0])
    edit(("append", h, em.Layers(R, NX, NZ, base["top"]).take(33), None))
    again = x.add_boundary(bigger)
    assert again != bx[0] and (again & 0xFFFF) == (bx[0] & 0xFFFF)
    with pytest.raises(Exception):
        x.read_boundary_particles(bx[0])
    bx[0] = again
    edit(("step", DT))
    edit(("delete", h, np.arange(model.slot(h).n) % 9 == 0))
    x.set_boundary_particles(bx[1], lid2)
    edit(("write", h, None, np.full((model.slot(h).n, 3), 0.01, F)))
    x.set_collider_state(cs_x, translation=box_at[1], body=BODY_FIXED)
    blob = x.snapshot()
    model.snapshot()

    y, _, by, cs_y = build(bigger, lid2)
    y.set_collider_state(cs_y, translation=box_at[1], body=BODY_FIXED)
    y.restore(blob)
    for _ in range(3):
        model.begin_step()
        x.step(DT)
        y.step(DT)
    for name, gx in em.read_world(x, h, False).items():
        assert em._first_diff(name, h, em.read_world(y, model.handles()[0], False)[name], gx) is None, name
    want = [bigger, lid2, (box + box_at[1]).astype(F), None]
    for k in range(4):
        px, vx = x.read_boundary_particles(bx[k])
        py, vy = y.read_boundary_particles(by[k])
        assert np.array_equal(px, py) and np.array_equal(vx, vy), "boundary %d" % k
        assert len(px) > 0 and (want[k] is None or np.array_equal(px, want[k])), "boundary %d holds another boundary's particles" % k
        if k != 3:   # the contact-sampled boundary changes size every step: its volumes are read by its own count
            assert all(np.array_equal(a, b) for a, b in zip(x.read_boundary(bx[k]), y.read_boundary(by[k])))
