"""Host model of the state a fluid particle carries through host edits between steps.  TEST INFRASTRUCTURE ONLY.

Written from the reference's rules, not from the engine: Fluid::add_particles (fluid.rs:126-150: appended at the end, default
volume), delete_particle_at_next_timestep (fluid.rs:71-76: a mark, counted once) applied by apply_particles_removal at the
next step in index order (fluid.rs:88-98, helper::filter_from_mask), the solver scratch that follows the same mask
(velocity_changes dfsph_solver.rs:526-561, pressures iisph_solver.rs:479-540: resized with zeros for new particles, then
filtered), the arena handles of add_fluid / remove_fluid (liquid_world.rs:161-178), and include/sph.h for what the reference
does not have (ids, replace_particles, snapshots).

The model does no physics.  After each step of a world the caller hands the world's positions, velocities, velocity_changes
and pressures to refresh(); ids, volumes, marks and the slot table stay the model's own bookkeeping.  Edits are
permutations, filters and splices, so a world and its model agree bit for bit after every edit (mismatches()).

Also here, because the CPU and the GPU tests share them: the seeded edit programs (make_program), their interpreter (apply_op)
and the comparisons (mismatches, step_mismatches, mass_mismatches, snapshot_bytes).
"""
import copy
import struct

import numpy as np

from . import ref64

F = np.float32
SOLVER_DFSPH, SOLVER_IISPH = 0, 1  # include/sph.h


def default_volume(particle_radius):
    r = F(particle_radius)
    return F(r * r * r * F(8.0 * 0.8))  # fluid.rs:110-120


class Slot:
    def __init__(self):
        self.alive, self.gen, self.density0 = False, 0, F(1000.0)
        self.memberships, self.filter, self.forces = 1, 0xFFFFFFFF, []
        self.clear()

    def clear(self):
        self.pos = np.zeros((0, 3), F)
        self.vel = np.zeros((0, 3), F)
        self.vc = np.zeros((0, 3), F)
        self.volume = np.zeros(0, F)
        self.pressure = np.zeros(0, F)
        self.id = np.zeros(0, np.uint32)
        self.pending = np.zeros(0, bool)

    ARRAYS = ("pos", "vel", "vc", "volume", "pressure", "id", "pending")

    @property
    def n(self):
        return len(self.pos)


def _f3(a):
    return np.ascontiguousarray(a, F).reshape(-1, 3).copy()


class EditModel:
    def __init__(self, particle_radius):
        self.volume0 = default_volume(particle_radius)
        self.slots = []

    # -- handles (slot | generation << 16) ---------------------------------------------------------------------------
    def slot(self, handle):
        k = handle & 0xFFFF
        if k >= len(self.slots) or not self.slots[k].alive or self.slots[k].gen != handle >> 16:
            raise KeyError("stale fluid handle %#x" % handle)
        return self.slots[k]

    def handles(self):
        return [k | s.gen << 16 for k, s in enumerate(self.slots) if s.alive]

    # -- edits -----------------------------------------------------------------------------------------------------------
    def add_fluid(self, positions, density0=1000.0, velocities=None, volumes=None, memberships=1, filter=0xFFFFFFFF):
        k = next((k for k, s in enumerate(self.slots) if not s.alive), len(self.slots))  # the first dead slot is reused
        if k == len(self.slots):
            self.slots.append(Slot())
            gen = 0
        else:
            gen = self.slots[k].gen + 1
            self.slots[k] = Slot()
        s = self.slots[k]
        s.alive, s.gen, s.density0, s.memberships, s.filter = True, gen, F(density0), memberships, filter
        s.pos = _f3(positions)
        n = s.n
        s.vel = np.zeros((n, 3), F) if velocities is None else _f3(velocities)
        s.vc = np.zeros((n, 3), F)
        s.volume = np.full(n, self.volume0, F) if volumes is None else np.array(volumes, F)
        s.pressure = np.zeros(n, F)
        s.id = np.arange(n, dtype=np.uint32)
        s.pending = np.zeros(n, bool)
        return k | gen << 16

    def push_force(self, handle, kind, params):
        self.slot(handle).forces.append((kind, list(params)))

    def next_id(self, s):
        """ids of appended particles count up from one past the largest id of the fluid, marked particles included"""
        return int(s.id.max()) + 1 if s.n else 0

    def append(self, handle, positions, velocities=None):
        s = self.slot(handle)
        p = _f3(positions)
        k = len(p)
        s.id = np.concatenate([s.id, (self.next_id(s) + np.arange(k)).astype(np.uint32)])
        s.pos = np.concatenate([s.pos, p])
        s.vel = np.concatenate([s.vel, np.zeros((k, 3), F) if velocities is None else _f3(velocities)])
        s.vc = np.concatenate([s.vc, np.zeros((k, 3), F)])            # dfsph_solver.rs:548
        s.volume = np.concatenate([s.volume, np.full(k, self.volume0, F)])
        s.pressure = np.concatenate([s.pressure, np.zeros(k, F)])     # iisph_solver.rs:499
        s.pending = np.concatenate([s.pending, np.zeros(k, bool)])

    def delete(self, handle, mask):
        s = self.slot(handle)
        mask = np.asarray(mask).astype(bool)
        if len(mask) != s.n:
            raise ValueError("mask length %d != particle count %d" % (len(mask), s.n))
        s.pending = s.pending | mask

    def write(self, handle, positions=None, velocities=None):
        s = self.slot(handle)
        for name, a in (("pos", positions), ("vel", velocities)):
            if a is None:
                continue
            a = _f3(a)
            if len(a) != s.n:  # the count before the marked particles go
                raise ValueError("length %d != particle count %d" % (len(a), s.n))
            setattr(s, name, a)

    def remove_fluid(self, handle):
        s = self.slot(handle)
        s.alive = False
        s.forces = []
        s.clear()

    def replace_particles(self, handle, positions, velocities=None, velocity_changes=None, ids=None):
        s = self.slot(handle)
        s.pos = _f3(positions)
        n = s.n
        s.vel = np.zeros((n, 3), F) if velocities is None else _f3(velocities)
        s.vc = np.zeros((n, 3), F) if velocity_changes is None else _f3(velocity_changes)
        s.id = np.arange(n, dtype=np.uint32) if ids is None else np.array(ids, np.uint32)
        s.volume = np.full(n, self.volume0, F)
        s.pressure = np.zeros(n, F)
        s.pending = np.zeros(n, bool)

    def set_ids(self, handle, ids):
        s = self.slot(handle)
        if len(ids) != s.n:
            raise ValueError("length %d != particle count %d" % (len(ids), s.n))
        s.id = np.array(ids, np.uint32)

    def filter_slot(self, s):
        """helper::filter_from_mask on everything a particle carries, in index order"""
        keep = ~s.pending
        for name in Slot.ARRAYS:
            setattr(s, name, getattr(s, name)[keep])

    def begin_step(self):
        for s in self.slots:
            if s.alive and s.pending.any():
                self.filter_slot(s)

    def snapshot(self):
        self.begin_step()  # taking a snapshot applies the marked deletions: part of the contract
        return [(s.alive, {name: getattr(s, name).copy() for name in Slot.ARRAYS}) for s in self.slots]

    def restore(self, snap):
        if len(snap) != len(self.slots) or any(a != s.alive for (a, _), s in zip(snap, self.slots)):
            raise ValueError("snapshot of a differently configured world")
        for (_, arrays), s in zip(snap, self.slots):
            for name in Slot.ARRAYS:
                setattr(s, name, arrays[name].copy())

    def refresh(self, handle, pos, vel, vc, pressure=None):
        """Take what a step computed from the world; everything else stays the model's own."""
        s = self.slot(handle)
        assert len(pos) == s.n
        s.pos, s.vel, s.vc = _f3(pos), _f3(vel), _f3(vc)
        if pressure is not None:
            s.pressure = np.array(pressure, F)

    def clone(self):
        return copy.deepcopy(self)


# ---- comparisons -----------------------------------------------------------------------------------------------------------
def _first_diff(name, handle, got, want):
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return "%s of fluid %#x: shape %s, the model has %s" % (name, handle, got.shape, want.shape)
    if np.array_equal(got, want):
        return None
    bad = np.nonzero((got != want).reshape(len(got), -1).any(axis=1))[0]
    k = int(bad[0])
    return "%s of fluid %#x: %d of %d particles differ, first at index %d: %s, the model has %s" % (
        name, handle, len(bad), len(got), k, got[k], want[k])


def read_world(world, handle, pressures):
    """Everything a world lets a caller read of a fluid's carried state."""
    if world.num_particles(handle) == 0:
        out = dict(pos=np.zeros((0, 3), F), vel=np.zeros((0, 3), F), vc=np.zeros((0, 3), F), id=np.zeros(0, np.uint32))
        if pressures:
            out["pressure"] = np.zeros(0, F)
        return out
    p, v = world.read_fluid(handle)
    out = dict(pos=p, vel=v, vc=world.debug(handle, "velocity_change"), id=world.read_ids(handle))
    if pressures:
        out["pressure"] = world.debug(handle, "pressure")
    return out


def stale_handles_refused(world, dead):
    out = []
    for h in dead:
        try:
            world.num_particles(h)
        except Exception:
            continue
        out.append("stale handle %#x still answers" % h)
    return out


def mismatches(world, model, pressures=False, dead=(), after_step=False):
    """What a world and its model disagree on, as text (empty: they agree bit for bit).  after_step: the step moved the
    particles, so only what an edit decides is compared: counts and ids."""
    out = []
    for h in model.handles():
        s = model.slot(h)
        try:
            n = world.num_particles(h)
        except Exception as e:
            out.append("fluid %#x of the model is refused by the world: %s" % (h, e))
            continue
        if n != s.n:
            out.append("fluid %#x has %d particles, the model has %d" % (h, n, s.n))
            continue
        got = read_world(world, h, pressures)
        for name in (("id",) if after_step else tuple(got)):
            d = _first_diff(name, h, got[name], getattr(s, name))
            if d:
                out.append(d)
    return out + stale_handles_refused(world, dead)


def snapshot_bytes(model, solver, dt, inv_dt):
    """The blob sph_world_snapshot_save writes (format version 1) for a single-GPU world holding the model's state, which
    must be a snapshot's: no marks pending.  Little-endian, in order: the header (magic "SPHS", version, solver, fluid slots,
    dt, inv_dt as float32, the slab planes INT32_MIN / INT32_MAX of an undivided world, the particle count, the blob's
    length); per slot its count, whether it is alive, its number of forces; the positions, velocities, velocity_changes,
    volumes, pressures and ids of every slot one after the other; per force a zero elasticity record (no rest pose)."""
    cols = (("pos", F), ("vel", F), ("vc", F), ("volume", F), ("pressure", F), ("id", np.uint32))
    body = b"".join(struct.pack("<QII", s.n, int(s.alive), len(s.forces)) for s in model.slots)
    body += b"".join(np.ascontiguousarray(getattr(s, name), t).tobytes() for name, t in cols for s in model.slots)
    body += b"".join(struct.pack("<QII", 0, 0, 0) for s in model.slots for _ in s.forces)
    head = "<IIIIffiiQQ"
    n = sum(s.n for s in model.slots)
    return struct.pack(head, 0x53485053, 1, solver, len(model.slots), dt, inv_dt, -2**31, 2**31 - 1, n,
                       struct.calcsize(head) + len(body)) + body


def snapshot_mismatches(blob, want):
    if blob == want:
        return []
    n = min(len(blob), len(want))
    differ = np.frombuffer(blob[:n], np.uint8) != np.frombuffer(want[:n], np.uint8)
    k = int(np.argmax(differ)) if differ.any() else n
    return ["the snapshot has %d bytes, the model's %d; they differ first at byte %d" % (len(blob), len(want), k)]


def refresh_from(world, model, pressures=False):
    for h in model.handles():
        got = read_world(world, h, pressures)
        model.refresh(h, got["pos"], got["vel"], got["vc"], got.get("pressure"))


def passes_of(model, h, boundaries, kw=0, kg=0):
    """ref64.Passes on the MODEL's positions, volumes, rest densities, fluid assignment and interaction groups, the fluids
    concatenated in slot order; boundaries: dicts with positions and optionally memberships / filter."""
    live = [s for s in model.slots if s.alive]
    P = np.concatenate([s.pos for s in live]) if live else np.zeros((0, 3), F)
    fid = np.concatenate([np.full(s.n, k) for k, s in enumerate(live)]).astype(np.int64)
    rho0 = np.concatenate([np.full(s.n, s.density0, F) for s in live])
    mass = np.concatenate([(s.volume * s.density0).astype(F) for s in live])  # fluid.rs:183-185
    BP = np.concatenate([b["positions"] for b in boundaries]).astype(F)
    bid = np.concatenate([np.full(len(b["positions"]), k) for k, b in enumerate(boundaries)]).astype(np.int64)
    fm = np.array([s.memberships for s in live], np.int64)
    ff = np.array([s.filter for s in live], np.int64)
    bm = np.array([b.get("memberships", 1) for b in boundaries], np.int64)
    bf = np.array([b.get("filter", 0xFFFFFFFF) for b in boundaries], np.int64)

    def test(m1, f1, m2, f2):  # interaction_groups.rs:20-79
        return ((m1 & f2) != 0) & ((m2 & f1) != 0)

    def allowed_ff(i, j):
        a, b = fid[i], fid[j]
        return (a == b) | test(fm[a], ff[a], fm[b], ff[b])

    def allowed_fb(i, j):
        a, b = fid[i], bid[j]
        return test(fm[a], ff[a], bm[b], bf[b])

    def allowed_bb(i, j):
        a, b = bid[i], bid[j]
        return (a == b) | test(bm[a], bf[a], bm[b], bf[b])

    return ref64.Passes(h, P, fid, rho0, mass, BP, bid, allowed_ff, allowed_fb, allowed_bb, kw=kw, kg=kg)


def mass_mismatches(ps, density, nf, nb, bvol, alpha=None):
    """The density pass of a step against ref64 on the model's state (ps = passes_of(model before the step)): contact counts
    exact, density (and alpha's denominator) within that pass's bound.  A volume or a fluid id that travelled with the
    wrong particle shows here and in no read-back.  density / nf / nb / alpha: the world's values, fluids concatenated in
    slot order; bvol: its boundary volumes."""
    from . import ref64_stages
    out = []
    for name, got, want in (("fluid", nf, ps.nf), ("boundary", nb, ps.nb)):
        bad = np.nonzero(np.asarray(got).astype(np.int64) != want)[0]
        if len(bad):
            out.append("%s contact counts differ at %d particles, first %d: %d, ref64 has %d" % (name, len(bad), bad[0], got[bad[0]], want[bad[0]]))
    r = ref64.ratio(density, ps.density(bvol), ref64.C_PASS["density"])
    r = np.where(ps.ambiguous(), 0.0, r)
    if len(r) and r.max() > 1.0:
        k = int(np.argmax(r))
        out.append("density exceeds its bound at %d particles, worst %d: |err| / bound = %.3g" % ((r > 1.0).sum(), k, r[k]))
    if alpha is not None:
        r, _ = ref64_stages.alpha_ratio(ps, np.asarray(alpha, F), bvol)
        if len(r) and r.max() > 1.0:
            out.append("alpha exceeds its bound: worst |err| / bound = %.3g" % r.max())
    return out


# ---- edit programs ---------------------------------------------------------------------------------------------------------
class Layers:
    """Where appended particles go: lattice layers of spacing 2r above the block, a fresh layer for every append."""

    def __init__(self, r, nx, nz, y0):
        self.r, self.nx, self.nz, self.y, self.used = r, nx, nz, y0, 0

    def take(self, k):
        assert k <= self.nx * self.nz
        i = np.arange(k)
        r = self.r
        p = np.stack([(2 * (i % self.nx) + 1) * r, np.full(k, self.y), (2 * (i // self.nx) + 1) * r], axis=1).astype(F)
        self.y += 2.2 * r
        return p


def make_program(seed, model, layers, dt, n_fill=10, host_only=True, per_volume=None):
    """About 40 concrete operations on the fluids of `model` (a throw-away copy follows the counts and the handles).
    Every program holds: delete -> step -> append with surviving ids above the shrunken count, a double mark, an append whose
    particle is marked before any step, writes on the host-staged and on the device path, an emptied fluid that is appended
    to later, set_ids, replace_particles, a snapshot taken with marks pending and restored two operations later, and (two
    fluids or more) a fluid that is not the last one removed and another count added into its slot.  host_only = False
    leaves out what only the engine has (ids, replace, snapshots, remove): the rest also runs on the oracle.
    Operations: ("step", dt) ("append", h, pos, vel) ("delete", h, mask) ("write", h, dpos, dvel: offsets added to the
    current values) ("remove", h) ("add", kwargs, forces) ("set_ids", h, perm) ("replace", h, perm) ("snapshot",)
    ("restore",) ("rebuild",): the place of a continuation check.  ("step", 0.0) follows the double mark."""
    rng = np.random.default_rng(seed)
    m = model.clone()
    ops, st = [], {}

    def emit(op):
        ops.append(op)
        if op[0] != "rebuild":
            apply_op(None, m, op, st)

    def pick():
        hs = [h for h in m.handles() if m.slot(h).n > 40]
        return hs[int(rng.integers(len(hs)))]

    def step():
        emit(("step", float(dt * (1.0, 2.0, 1.0 / 3.0)[int(rng.integers(3))])))

    def append(h, k, vel):
        p = layers.take(k)
        emit(("append", h, p, rng.normal(0, 0.2, p.shape).astype(F) if vel else None))

    def random_mask(h, frac=0.05):
        return rng.random(m.slot(h).n) < frac

    def delete_step_append():
        h = pick()
        mask = np.zeros(m.slot(h).n, bool)
        mask[:30] = True  # the survivors keep ids at and above the shrunken count
        emit(("delete", h, mask))
        step()
        append(h, 33, True)
        emit(("rebuild",))

    def double_mark():
        h = pick()
        mask = random_mask(h)
        emit(("delete", h, mask))
        again = mask.copy()
        again[int(rng.integers(len(mask)))] = True
        emit(("delete", h, again))
        if host_only:  # a step of no time applies the marks and computes nothing: what the step's filter did is compared in full
            emit(("step", 0.0))

    def append_then_mark():
        h = pick()
        append(h, 1, False)
        mask = np.zeros(m.slot(h).n, bool)
        mask[-1] = True
        emit(("delete", h, mask))
        emit(("append", h, np.zeros((0, 3), F), None))

    def write(h, pos, vel):
        n = m.slot(h).n
        emit(("write", h, (rng.uniform(-0.05, 0.05, (n, 3)) * layers.r).astype(F) if pos else None,
              rng.normal(0, 0.05, (n, 3)).astype(F) if vel else None))

    def staged_write():
        h = pick()
        append(h, 33, False)
        write(h, True, True)

    def device_writes():
        step()
        write(pick(), True, False)
        step()
        write(pick(), False, True)

    def empty_and_refill():
        hs = m.handles()
        h = hs[-1] if len(hs) > 1 else hs[0]
        emit(("delete", h, np.ones(m.slot(h).n, bool)))
        step()
        step()
        append(h, 33, True)
        append(h, 33, False)

    def set_ids():
        h = pick()
        emit(("set_ids", h, rng.permutation(m.slot(h).n)))

    def replace():
        hs = [h for h in m.handles() if m.slot(h).n > 40 and h != per_volume] or [pick()]
        h = hs[int(rng.integers(len(hs)))]
        emit(("replace", h, rng.permutation(m.slot(h).n)))
        step()

    def snapshot_restore():
        h = pick()
        emit(("delete", h, random_mask(h)))
        emit(("snapshot",))
        step()
        write(pick(), True, True)
        emit(("restore",))

    def remove_and_add():
        hs = m.handles()
        if len(hs) < 2:
            return
        h = hs[len(hs) // 2 - (len(hs) == 2)]  # the middle fluid; of two, the first
        s = m.slot(h)
        n = s.n // 2 + 7
        kwargs = dict(positions=s.pos[:n] + F(0.01 * layers.r), density0=float(s.density0), velocities=s.vel[:n].copy(),
                      volumes=(m.volume0 * rng.uniform(0.9, 1.1, n)).astype(F), memberships=s.memberships, filter=s.filter)
        forces = list(s.forces)
        emit(("delete", h, random_mask(h)))  # removed with marks pending
        emit(("remove", h))
        step()
        emit(("add", kwargs, forces))

    motifs = [delete_step_append, double_mark, append_then_mark, staged_write, device_writes, empty_and_refill]
    if host_only:
        motifs += [set_ids, replace, snapshot_restore, remove_and_add]
    order = rng.permutation(len(motifs)).tolist()
    if len(m.handles()) == 1:  # the only fluid is emptied last, so that the other edits meet the whole block
        order.remove(motifs.index(empty_and_refill))
        order.append(motifs.index(empty_and_refill))
    fill = sorted(rng.integers(0, len(motifs) + 1, n_fill).tolist())
    marks = set(rng.choice(len(motifs), 2, replace=False).tolist())
    for k, o in enumerate(order):
        for _ in range(fill.count(k)):
            step()
        motifs[o]()
        if k in marks:
            emit(("rebuild",))
    for _ in range(fill.count(len(motifs))):
        step()
    emit(("rebuild",))
    return ops


def apply_op(world, model, op, state, pressures=False):
    """Apply one operation to a world (None: the model alone) and to its model.  `state` carries the snapshot between its
    two operations and the handles that died.  A step refreshes the model from the world after comparing what the step must
    not have changed: counts and ids.  What a delete applied INSIDE a step did to positions, velocities, vc and pressures is
    therefore compared only where marks are applied and nothing is computed: at a step of dt = 0 (the step's own path:
    the marks go, the state is uploaded, the solver does not run) and at a snapshot, whose bytes must be snapshot_bytes of
    the model.  pressures: the world is an IISPH one, whose pressures are carried.  Returns the mismatches after the
    operation."""
    kind = op[0]
    dead = state.setdefault("dead", [])
    after_step, out = False, []
    if kind == "step":
        model.begin_step()
        if world is not None:
            world.step(op[1])
        after_step = op[1] > 0
    elif kind == "append":
        model.append(op[1], op[2], op[3])
        if world is not None:
            world.append_particles(op[1], op[2], op[3])
    elif kind == "delete":
        model.delete(op[1], op[2])
        if world is not None:
            world.delete_particles(op[1], op[2])
    elif kind == "write":
        s = model.slot(op[1])
        p = None if op[2] is None else (s.pos + op[2]).astype(F)
        v = None if op[3] is None else (s.vel + op[3]).astype(F)
        model.write(op[1], p, v)
        if world is not None:
            world.write_fluid(op[1], p, v)
    elif kind == "remove":
        model.remove_fluid(op[1])
        dead.append(op[1])
        if world is not None:
            world.remove_fluid(op[1])
    elif kind == "add":
        h = model.add_fluid(**op[1])
        for f in op[2]:
            model.push_force(h, *f)
        if world is not None:
            hw = world.add_fluid(op[1]["positions"], **{k: v for k, v in op[1].items() if k != "positions"})
            for f in op[2]:
                world.push_force(hw, *f)
            if hw != h:
                return ["add_fluid returned the handle %#x, the model %#x" % (hw, h)]
    elif kind == "set_ids":
        ids = model.slot(op[1]).id[op[2]]
        model.set_ids(op[1], ids)
        if world is not None:
            world.set_ids(op[1], ids)
    elif kind == "replace":
        s, perm = model.slot(op[1]), op[2]
        args = (s.pos[perm], s.vel[perm], s.vc[perm], s.id[perm])
        model.replace_particles(op[1], *args)
        if world is not None:
            world.replace_particles(op[1], *args)
    elif kind == "snapshot":
        state["model_snapshot"] = model.snapshot()
        if world is not None:
            blob = state["world_snapshot"] = world.snapshot()
            if isinstance(blob, bytes):  # an engine's blob; a stand-in world built on a model hands back the model's snapshot
                dt, inv_dt = struct.unpack_from("<ff", blob, 16)  # the lagging timestep is the world's, not the model's
                out = snapshot_mismatches(blob, snapshot_bytes(model, SOLVER_IISPH if pressures else SOLVER_DFSPH, dt, inv_dt))
    elif kind == "restore":
        model.restore(state["model_snapshot"])
        if world is not None:
            world.restore(state["world_snapshot"])
    else:
        raise ValueError(kind)
    if world is None:
        return []
    out += mismatches(world, model, pressures, dead, after_step)
    if after_step and not out:
        refresh_from(world, model, pressures)
    return out


def has_collision_pattern(ops, model):
    """True if the program appends to a fluid after a delete and a step, while a survivor's id is at or above the shrunken
    count: where ids numbered from the count would repeat."""
    m = model.clone()
    shrunk, st = set(), {}
    for op in ops:
        if op[0] == "rebuild":
            continue
        before = {h: m.slot(h).n for h in m.handles()}
        if op[0] == "append" and len(op[2]) and op[1] in shrunk:
            s = m.slot(op[1])
            if s.n and int(s.id.max()) >= s.n:
                return True
        apply_op(None, m, op, st)
        if op[0] == "step":
            shrunk |= {h for h in m.handles() if h in before and m.slot(h).n < before[h]}
    return False
