"""oracle/edit_model.py without a GPU: the model against the CPU oracle on the operations the oracle has, and the checker
against mutants.  Each mutant is one plausible splice bug of an engine; the programs and the comparison functions are the
ones tests/test_gpu_edits.py runs, with the unmutated model (and a stand-in step) in the engine's place, so a mutant that is
not flagged here would not be flagged on the GPU either."""
import struct

import numpy as np
import pytest

import test_gpu_edits as ge
from oracle import edit_model as em
from oracle.oracle import OracleWorld

F = np.float32


class ModelWorld:
    """An EditModel behind the calls of a LiquidWorld.  step() is not physics: it moves every carried quantity by a
    particle-specific amount, so that a quantity attached to the wrong particle reads differently."""

    def __init__(self, model, boundaries):
        self.m, self.boundaries, self.h = model, boundaries, F(4 * ge.R)
        self.scratch = {}

    def add_fluid(self, positions, **kw):
        return self.m.add_fluid(positions, **kw)

    def push_force(self, h, kind, params):
        self.m.push_force(h, kind, params)

    def add_boundary(self, positions):
        return 0

    def step(self, dt):
        m = self.m
        m.begin_step()
        if not dt > 0:
            return
        if any(s.alive and s.n for s in m.slots):
            ps = em.passes_of(m, self.h, self.boundaries)
            self.bvol = (1.0 / ps.boundary_volume_sum().value).astype(F)
            self.scratch = dict(density=ps.density(self.bvol).value.astype(F), num_fluid_contacts=ps.nf.astype(F),
                                num_boundary_contacts=ps.nb.astype(F))
        for s in m.slots:
            if s.alive:
                s.vc = (F(0.5) * s.vc + F(dt) * s.vel + F(1e-3) * s.pos).astype(F)
                s.vel = (s.vel + s.vc).astype(F)
                s.pos = (s.pos + F(dt) * s.vel).astype(F)
                s.pressure = (np.abs(s.pos.sum(axis=1)) * F(100.0) + F(1.0)).astype(F)

    def num_particles(self, h):
        return self.m.slot(h).n

    def read_fluid(self, h):
        s = self.m.slot(h)
        return s.pos.copy(), s.vel.copy()

    def read_ids(self, h):
        return self.m.slot(h).id.copy()

    def debug(self, h, what):
        s = self.m.slot(h)
        if what in ("velocity_change", "pressure"):
            return (s.vc if what == "velocity_change" else s.pressure).copy()
        live = [x for x in self.m.slots if x.alive]
        at = sum(x.n for x in live[:live.index(s)])
        return self.scratch[what][at:at + s.n]

    def append_particles(self, h, p, v=None):
        self.m.append(h, p, v)

    def delete_particles(self, h, mask):
        self.m.delete(h, mask)

    def write_fluid(self, h, positions=None, velocities=None):
        self.m.write(h, positions, velocities)

    def remove_fluid(self, h):
        self.m.remove_fluid(h)

    def set_ids(self, h, ids):
        self.m.set_ids(h, ids)

    def replace_particles(self, h, *args):
        self.m.replace_particles(h, *args)

    def snapshot(self):
        return self.m.snapshot()

    def restore(self, blob):
        self.m.restore(blob)


# ---- mutants ---------------------------------------------------------------------------------------------------------------
class AppendInheritsVc(em.EditModel):
    """appended particles take the velocity_changes of the slots they land in (those of the next fluid, or stale ones)"""

    def append(self, h, p, v=None):
        s = self.slot(h)
        k = len(np.reshape(p, (-1, 3)))
        live = [x for x in self.slots if x.alive and x.n]
        src = live[(live.index(s) + 1) % len(live)].vc if s in live else np.ones((1, 3), F)
        super().append(h, p, v)
        if k:
            s.vc[-k:] = np.resize(src, (k, 3))


class VcNotFiltered(em.EditModel):
    def filter_slot(self, s):
        vc = s.vc.copy()
        super().filter_slot(s)
        s.vc = vc[:s.n]


class PressureMaskShifted(em.EditModel):
    def filter_slot(self, s):
        pr = s.pressure[~np.roll(s.pending, 1)]
        super().filter_slot(s)
        s.pressure = np.resize(pr, s.n) if len(pr) else np.zeros(s.n, F)


class DeleteImmediately(em.EditModel):
    def delete(self, h, mask):
        super().delete(h, mask)
        self.filter_slot(self.slot(h))


class DoubleMarkCountedTwice(em.EditModel):
    """a counter of marks that counts a particle marked twice two times, and a removal that trusts it for the new count"""

    def delete(self, h, mask):
        s = self.slot(h)
        s.count = getattr(s, "count", 0) + int(np.asarray(mask).astype(bool).sum())
        super().delete(h, mask)

    def filter_slot(self, s):
        kept = max(s.n - getattr(s, "count", 0), 0)
        super().filter_slot(s)
        for name in em.Slot.ARRAYS:
            setattr(s, name, getattr(s, name)[:kept])
        s.count = 0


class AppendDoesNotShiftNextFluid(em.EditModel):
    """an append into fluid k leaves the ids and pressures of fluid k + 1 where they were in the world's arrays"""

    def append(self, h, p, v=None):
        s = self.slot(h)
        k = len(np.reshape(p, (-1, 3)))
        super().append(h, p, v)
        live = [x for x in self.slots if x.alive]
        nxt = live[live.index(s) + 1:]
        if k and nxt and nxt[0].n:
            t = nxt[0]
            t.id = np.roll(t.id, k)
            t.pressure = np.roll(t.pressure, k)


class VolumesNotFiltered(em.EditModel):
    def filter_slot(self, s):
        vol = s.volume.copy()
        super().filter_slot(s)
        s.volume = vol[:s.n]


class WritePositionsOverwritesVelocities(em.EditModel):
    def write(self, h, positions=None, velocities=None):
        super().write(h, positions, velocities)
        if positions is not None and velocities is None:
            self.slot(h).vel[:] = 0


class RemovedSlotNotReused(em.EditModel):
    def add_fluid(self, positions, **kw):
        dead = [s for s in self.slots if not s.alive]
        for s in dead:
            s.alive = True
        h = super().add_fluid(positions, **kw)
        for s in dead:
            s.alive = False
        return h


class IdsFromTheCount(em.EditModel):
    """the rule this project had: an appended particle's id is the fluid's count"""

    def next_id(self, s):
        return s.n


MUTANTS = {"appended particles inherit the vc of the slot they land in": AppendInheritsVc,
           "vc not filtered on delete": VcNotFiltered,
           "pressures filtered with the mask shifted by one": PressureMaskShifted,
           "deletes applied at the call instead of at the next step": DeleteImmediately,
           "a double mark counted twice": DoubleMarkCountedTwice,
           "append into fluid k not shifting fluid k+1's ids / pressures": AppendDoesNotShiftNextFluid,
           "volumes not filtered": VolumesNotFiltered,
           "write of positions only also overwriting velocities": WritePositionsOverwritesVelocities,
           "a removed slot not reused": RemovedSlotNotReused,
           "ids numbered from the count": IdsFromTheCount}


def run(scene, ops, model_class):
    """The program with the unmutated model as the world and `model_class` as the model under the GPU test's comparisons:
    every read-back after every operation, and the mass check at each continuation point and at the end.  Returns the
    first mismatches."""
    world, model = ModelWorld(em.EditModel(ge.R), scene["boundaries"]), model_class(ge.R)
    ge.populate(world, model, scene)
    state = {}

    def mass():
        model.begin_step()
        ps = em.passes_of(model, world.h, scene["boundaries"])
        world.step(ge.DT)
        live = [h for h in world.m.handles() if world.m.slot(h).n]
        cat = lambda what: np.concatenate([world.debug(h, what) for h in live])  # noqa: E731
        bad = em.mass_mismatches(ps, cat("density"), cat("num_fluid_contacts"), cat("num_boundary_contacts"), world.bvol)
        bad = bad or em.mismatches(world, model, True, after_step=True)
        if not bad:
            em.refresh_from(world, model, True)
        return bad

    for k, op in enumerate(ops):
        try:
            bad = mass() if op[0] == "rebuild" else em.apply_op(world, model, op, state, pressures=True)
        except (KeyError, ValueError, IndexError) as e:
            bad = ["the model refuses operation %d %s: %s" % (k, op[0], e)]
        if bad:
            return ["operation %d %s: %s" % (k, op[0], b) for b in bad]
    return mass()


SCENES = ("dfsph1", "dfsph3", "iisph2")


@pytest.fixture(scope="module")
def all_programs():
    return {name: ge.programs(name) for name in SCENES}


def test_the_programs_hold_what_they_must(all_programs):
    for name, (scene, progs) in all_programs.items():
        model = em.EditModel(ge.R)
        ge.populate(None, model, scene)
        assert len(progs) >= 3
        for ops in progs:
            kinds = [op[0] for op in ops]
            assert 35 <= len(kinds) <= 70
            assert em.has_collision_pattern(ops, model)
            assert kinds.count("rebuild") >= 4 and kinds[-1] == "rebuild"
            for need in ("step", "append", "delete", "write", "set_ids", "replace", "snapshot", "restore") + (("remove", "add") if name != "dfsph1" else ()):
                assert need in kinds, (name, need)
            assert any(op[0] == "append" and len(op[2]) == k for op in ops for k in (0,)) and any(op[0] == "append" and len(op[2]) == 1 for op in ops)
            assert any(op[0] == "write" and op[3] is None for op in ops) and any(op[0] == "write" and op[2] is None for op in ops)


def test_the_unmutated_model_agrees_with_itself(all_programs):
    for name, (scene, progs) in all_programs.items():
        for ops in progs:
            assert run(scene, ops, em.EditModel) == []


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutant_is_caught(mutant, all_programs):
    caught = []
    for name, (scene, progs) in all_programs.items():
        for k, ops in enumerate(progs):
            bad = run(scene, ops, MUTANTS[mutant])
            if bad:
                caught.append("%s program %d, %s" % (name, k, bad[0]))
    assert caught, "no program flags the mutant: " + mutant
    print("caught %r in %d of 9 programs; first: %s" % (mutant, len(caught), caught[0]))


def test_ids_from_the_count_repeat_a_survivors_id(all_programs):
    scene, progs = all_programs["dfsph1"]
    model = IdsFromTheCount(ge.R)
    ge.populate(None, model, scene)
    state, repeated = {}, False
    for op in progs[0]:
        if op[0] != "rebuild":
            em.apply_op(None, model, op, state)
        repeated |= any(len(np.unique(model.slot(h).id)) < model.slot(h).n for h in model.handles())
    assert repeated


def test_snapshot_bytes_lay_out_the_model_in_slot_order():
    """em.snapshot_bytes, which the GPU programs compare every world's snapshot with: the 48-byte header, a 16-byte record
    per slot (a removed one included), the six columns each over all slots, a 16-byte zero record per force."""
    scene = ge.make_scene("dfsph3")
    model = em.EditModel(ge.R)
    ge.populate(None, model, scene)
    h0, h1, h2 = model.handles()
    model.delete(h2, np.arange(model.slot(h2).n) % 3 == 0)
    model.remove_fluid(h1)
    model.snapshot()
    blob = em.snapshot_bytes(model, em.SOLVER_DFSPH, 0.004, 250.0)
    n = [s.n for s in model.slots]
    assert n[1] == 0 and 0 < n[2] < len(scene["fluids"][2]["positions"])   # the marks went with the snapshot
    head = struct.unpack_from("<IIIIffiiQQ", blob)
    assert head == (0x53485053, 1, em.SOLVER_DFSPH, 3, F(0.004), 250.0, -2**31, 2**31 - 1, sum(n), len(blob))
    assert [struct.unpack_from("<QII", blob, 48 + 16 * k) for k in range(3)] == [(n[0], 1, 1), (0, 0, 0), (n[2], 1, 1)]
    at, N = 48 + 16 * 3, sum(n)
    for name, width, t in (("pos", 3, F), ("vel", 3, F), ("vc", 3, F), ("volume", 1, F), ("pressure", 1, F), ("id", 1, np.uint32)):
        col = np.frombuffer(blob, t, width * N, at)
        assert np.array_equal(col, np.concatenate([getattr(s, name).reshape(-1) for s in model.slots])), name
        at += 4 * width * N
    assert blob[at:] == bytes(16 * 2)   # the forces of slots 0 and 2; the removed slot has none


# ---- the model against the CPU oracle --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCENES)
def test_model_counts_and_untouched_particles_match_the_oracle(name):
    """The same seeded program on the oracle and on the model: counts equal after every operation; between two steps the
    oracle's positions and velocities are the model's (refreshed from the oracle at every step) bit for bit, which pins
    append at the end, delete in index order at the next step, a mark counted once, and both halves of write."""
    scene, progs = ge.programs(name, host_only=False, seeds=(1,), n_fill=2)
    cpu = OracleWorld(ge.R, 2.0, solver=scene["solver"])
    model = em.EditModel(ge.R)
    ge.populate(None, model, scene)
    for f in scene["fluids"]:
        h = cpu.add_fluid(f["positions"], density0=f["density0"], velocities=f.get("velocities"), volumes=f.get("volumes"),
                          memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF))
        for force in f["forces"]:
            cpu.push_force(h, *force)
    for b in scene["boundaries"]:
        cpu.add_boundary(b["positions"])
    cpu.force_iterations(1, 2)
    state = {}
    for op in progs[0]:
        if op[0] == "rebuild":
            continue
        if op[0] == "write":   # the offsets are added to the model's values, which are the oracle's
            s = model.slot(op[1])
            cpu.write_fluid(op[1], None if op[2] is None else (s.pos + op[2]).astype(F), None if op[3] is None else (s.vel + op[3]).astype(F))
        else:
            ge._oracle_apply(cpu, op)
        em.apply_op(None, model, op, state)
        for h in model.handles():
            s = model.slot(h)
            assert cpu.num_particles(h) == s.n, op[0]
            if not s.n:
                continue
            p, v = cpu.read_fluid(h)
            if op[0] == "step":
                model.refresh(h, p, v, cpu.debug(h, "velocity_change"))
            else:
                assert np.array_equal(p, s.pos) and np.array_equal(v, s.vel), op[0]
