"""What sph_fluid_push_host_force2 hands a user's NonPressureForce::solve, captured inside the callback and checked against
the float64 reference (oracle/ref64_context.py): every materialised contact's indices, weight and gradient, the particle and
boundary views, the accelerations on entry (within the reference's bound of gravity plus the force pushed before, and bit
for bit against a twin world whose callback adds the same without contacts or boundaries) and the plugin's additions
after the step, on its own fluid's rows only.  Each case prints one CTX64 line with the worst |err| / bound and the exclusions."""
import json

import numpy as np
import pytest

from oracle import ref64
from oracle import ref64_context as X
from oracle import ref64_stages as S
from salva_b200 import BODY_NONE, DFSPHSolver, DynamicContactSampling, IISPHSolver, LiquidWorld, StaticSampling, scenes
from salva_b200.liquid_world import Ball, Cuboid, Poly6Kernel, SpikyKernel, ViscosityKernel

pytestmark = pytest.mark.gpu

F = np.float32
K = {1: Poly6Kernel, 2: SpikyKernel, 3: ViscosityKernel}
GRAVITY = (0.0, -9.81, 0.0)
ART = (1.0, 0.0, 1.0, 0.0, 10.0)   # ArtificialViscosity (cf, cb, alpha, beta, cs) pushed before the host forces


def _maker(kd=0, kg=0, iisph=False):
    def make():
        cls = IISPHSolver if iisph else DFSPHSolver
        return LiquidWorld(cls(K[kd], K[kg]) if kd else cls(), particle_radius=S.R, smoothing_factor=2.0)
    return make


class Rig:
    """A world with host forces and its twin, driven through the same edits; per slot what the fluids hold."""

    def __init__(self, scene, make, host, pre=(), flags=(True, True), kw=0, kg=0, iisph=False):
        self.w, self.t = make(), make()
        self.kw, self.kg, self.iisph, self.flags, self.pre = kw, kg, iisph, flags, pre
        self.fl, self.bd, self.calls, self.tcalls, self.rep = {}, {}, [], [], X.Report()
        self.host = {}
        for f in scene["fluids"]:
            self.add_fluid(f)
        for b in scene["boundaries"]:
            self.add_boundary(b)
        for slot, salt in host:
            self.push_host(slot, salt)

    def add_fluid(self, f):
        hs = []
        for w in (self.w, self.t):
            (h,), _ = S.populate(w, dict(fluids=[f], boundaries=[]), [scenes.artificial_viscosity(*ART)] if self.pre else ())
            hs.append(h)
        n = self.w.num_particles(hs[0])
        vdef = F(F(S.R) * F(S.R) * F(S.R) * F(8.0 * 0.8))
        vol = np.full(n, vdef, F)
        if f.get("volumes") is not None:
            vol[:len(f["volumes"])] = f["volumes"]
        slot = hs[0] & 0xFFFF
        assert hs[1] & 0xFFFF == slot
        self.fl[slot] = dict(h=hs[0], th=hs[1], density0=f["density0"], memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF),
                             volumes=vol, keep=np.ones(n, bool) if "deleted" not in f else np.r_[np.ones(len(f["positions"]), bool),
                                                                                              np.zeros(len(f["deleted"]), bool)])
        return slot

    def add_boundary(self, b):
        hs = [w.add_boundary(b["positions"], velocities=b.get("velocities"), memberships=b.get("memberships", 1),
                             filter=b.get("filter", 0xFFFFFFFF), want_forces=b.get("want_forces", False)) for w in (self.w, self.t)]
        slot = hs[0] & 0xFFFF
        self.bd[slot] = dict(h=hs[0], th=hs[1], memberships=b.get("memberships", 1), filter=b.get("filter", 0xFFFFFFFF))
        return slot

    def push_host(self, slot, salt):
        """The plugin under test on the world; on the twin the same additions through the callback without contacts or
        boundaries, so that both stay on one trajectory, and the twin's callback keeps what it was handed."""
        def solve(ctx):
            self.calls.append((slot, salt, X.capture(ctx)))
            ctx.accelerations += X.pattern(len(ctx.positions), slot, salt)

        def twin(dt, inv_dt, h, pos, vel, dens, acc):
            self.tcalls.append((slot, salt, acc.copy()))
            acc += X.pattern(len(acc), slot, salt)
        self.w.push_host_force2(self.fl[slot]["h"], solve, contacts=self.flags[0], boundaries=self.flags[1])
        self.t.push_host_force(self.fl[slot]["th"], twin)
        self.host.setdefault(slot, []).append(salt)

    def delete(self, slot, mask):
        for w, h in ((self.w, self.fl[slot]["h"]), (self.t, self.fl[slot]["th"])):
            w.delete_particles(h, mask)
        self.fl[slot]["keep"] = ~np.asarray(mask, bool)

    def append(self, slot, pos):
        for w, h in ((self.w, self.fl[slot]["h"]), (self.t, self.fl[slot]["th"])):
            w.append_particles(h, pos)
        d = self.fl[slot]
        d["volumes"] = np.r_[d["volumes"], np.full(len(pos), F(F(S.R) * F(S.R) * F(S.R) * F(8.0 * 0.8)), F)].astype(F)
        d["keep"] = np.r_[d["keep"], np.ones(len(pos), bool)]

    def remove_fluid(self, slot):
        d = self.fl.pop(slot)
        self.w.remove_fluid(d["h"])
        self.t.remove_fluid(d["th"])
        self.host.pop(slot, None)

    def remove_boundary(self, slot):
        d = self.bd.pop(slot)
        self.w.remove_boundary(d["h"])
        self.t.remove_boundary(d["th"])

    def _fluid_slots(self):
        return range(max(self.fl) + 1) if self.fl else range(0)

    def step(self, dt=S.DT, gravity=GRAVITY, iters=None):
        pre = {}
        for s, d in self.fl.items():
            P, V = self.w.read_fluid(d["h"])
            k = d["keep"]
            pre[s] = (P[k], V[k], d["volumes"][k])
        self._pre_v = {s: p[1] for s, p in pre.items()}
        for s, d in self.fl.items():   # the step applies the pending deletes
            d["volumes"], d["keep"] = d["volumes"][d["keep"]], np.ones(int(d["keep"].sum()), bool)
        self.calls, self.tcalls = [], []
        for w in (self.w, self.t):
            if iters is not None:
                w.force_iterations(*iters)
            w.step(dt, gravity)
        self._check(pre, gravity)

    def _check(self, pre, gravity):
        w, t = self.w, self.t
        nslot = len(self._fluid_slots())
        empty3, empty1 = np.zeros((0, 3), F), np.zeros(0, F)
        post = {s: dict(V=w.read_fluid(d["h"])[1], dens=w.debug(d["h"], "density"), acc=w.debug(d["h"], "acceleration"),
                        tacc=t.debug(d["th"], "acceleration"), nf=w.debug(d["h"], "num_fluid_contacts").astype(np.int64),
                        nb=w.debug(d["h"], "num_boundary_contacts").astype(np.int64)) for s, d in self.fl.items()}
        nb_slots = max(self.bd) + 1 if self.bd else 0
        bst = []
        for b in range(nb_slots):
            if b in self.bd:
                P, V = w.read_boundary_particles(self.bd[b]["h"])
                bst.append(dict(positions=P, velocities=V, volumes=w.read_boundary(self.bd[b]["h"])[0], **{k: self.bd[b][k] for k in ("memberships", "filter")}))
            else:
                bst.append(dict(positions=empty3, velocities=empty3, volumes=empty1))
        fst = [dict(positions=pre[s][0], volumes=pre[s][2], **{k: self.fl[s][k] for k in ("density0", "memberships", "filter")})
               if s in self.fl else dict(positions=empty3, volumes=empty1, density0=1000.0) for s in range(nslot)]
        st = X.State(S.R, fst, bst, self.kw, self.kg)
        # each host force is called exactly once per step, empty fluids included, in push order
        want = sorted((s, salt) for s, salts in self.host.items() for salt in salts)
        assert sorted((s, salt) for s, salt, _ in self.calls) == want and sorted((s, salt) for s, salt, _ in self.tcalls) == want
        tentry = {(s, salt): a for s, salt, a in self.tcalls}
        last = {}
        for s, salt, cap in self.calls:
            ex = dict(velocities=pre[s][1] if self.iisph else post[s]["V"], densities=post[s]["dens"], volumes=pre[s][2],
                      acc_in=tentry[(s, salt)], counts_ff=post[s]["nf"], counts_fb=post[s]["nb"], handle=self.fl[s]["h"],
                      density0=self.fl[s]["density0"], particle_radius=S.R, h=w.h, contacts=self.flags[0], boundaries=self.flags[1],
                      boundary_n=[len(b["positions"]) for b in bst])
            X.check(cap, st, s, ex, self.rep)
            if s in last:   # a second host force on the fluid sees the first one's additions
                prev_salt, prev = last[s]
                self.rep.exact("acc_chain", [s] if len(X._bitwise_rows(cap["accelerations"], prev["accelerations"] +
                                                                      X.pattern(prev["n"], s, prev_salt))) else [])
            last[s] = (salt, cap)
            if self.pre and salt == 0 and cap["n"]:
                self._acc_in_ref64(st, cap, s, post, bst, gravity)
        after = [post[k]["acc"] if k in post else empty3 for k in range(nslot)]
        for s, (salt, cap) in last.items():
            X.check_acc_out(after, [post[k]["tacc"] if k in post else empty3 for k in range(nslot)], cap["accelerations"],
                            X.pattern(cap["n"], s, salt), s, self.rep)

    def _acc_in_ref64(self, st, cap, s, post, bst, gravity):
        """The entry accelerations against gravity plus the ArtificialViscosity pushed before, on the velocities and densities
        the force read."""
        ps = st.passes()
        slots = range(len(st.fluids))
        V = np.concatenate([np.zeros((0, 3), F) if k not in post else self._pre_v[k] if self.iisph else post[k]["V"] for k in slots]).astype(F)
        D = np.concatenate([post[k]["dens"] if k in post else np.zeros(0, F) for k in slots]).astype(F)
        bvel = np.concatenate([b["velocities"] for b in bst]).astype(F) if bst else np.zeros((0, 3), F)
        bvol = np.concatenate([b["volumes"] for b in bst]).astype(F) if bst else np.zeros(0, F)
        ref, amb = ps.artificial(V, D, *ART[:2], ART[2], ART[3], ART[4], bvel, bvol)
        g = np.asarray(gravity, F).astype(np.float64)
        ref = ref64.Ref(ref.value + g, ref.A + np.abs(g), ref.K, ref.n + 1)
        fo = st.offsets(st.fluids)
        rows = slice(fo[s], fo[s + 1])
        r = ref64.ratio(cap["accelerations"], ref64.Ref(ref.value[rows], ref.A[rows], ref.K[rows], ref.n[rows]), ref64.C_PASS["artificial"])
        ex = (amb | ps.ambiguous())[rows]
        self.rep.ratio("acc_in_ref64", np.where(ex, 0.0, r.max(axis=1)))
        self.rep.excluded["acc_in_ref64"] = self.rep.excluded.get("acc_in_ref64", 0) + int(ex.sum())

    def finish(self, case):
        print("\nCTX64 %s" % json.dumps(dict(case=case, worst={k: round(v, 5) for k, v in self.rep.worst.items()},
                                             excluded={k: v for k, v in self.rep.excluded.items() if v})))
        for w in (self.w, self.t):
            w.close()
        assert not self.rep.flagged(), self.rep.flagged()
        return self.rep


def _run(case, scene, steps=2, make=None, host=None, pre=True, **kw):
    host = [(k, 0) for k in range(len(scene["fluids"]))] + [(0, 1)] if host is None else host
    rig = Rig(scene, make or _maker(kw.get("kw", 0), kw.get("kg", 0), kw.get("iisph", False)), host, pre=pre, **kw)
    for _ in range(steps):
        rig.step()
    return rig.finish(case)


CTX_SCENES = ("block", "pairs", "volumes", "two_fluids", "tail1", "tail33")


@pytest.mark.parametrize("name", CTX_SCENES)
def test_host_force_ctx_matches_ref64(name):
    rep = _run(name, S.SCENES[name]())
    assert {"ff_gradient", "fb_gradient", "ff_weight", "acc_in_ref64", "boundary_volume"} <= set(rep.worst)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids"])
@pytest.mark.parametrize("kd,kg", [(1, 2), (3, 1)], ids=["poly6+spiky", "viscosity+poly6"])
def test_host_force_ctx_matches_ref64_with_generic_kernels(name, kd, kg):
    # the viscosity kernel's W ~ h / 2r at the pairs scene's near-coincident pairs: the first step blows them apart
    _run("%s/%d%d" % (name, kd, kg), S.SCENES[name](), steps=1 if (name, kd) == ("pairs", 3) else 2, kw=kd, kg=kg)


@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids"])
def test_host_force_ctx_matches_ref64_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _run(name + "/xysub2", S.SCENES[name]())


@pytest.mark.parametrize("name", ["block", "two_fluids"])
def test_host_force_ctx_matches_ref64_under_iisph(name):
    _run(name + "/iisph", S.SCENES[name](), iisph=True)


def test_host_force_ctx_on_sixteen_fluids():
    """Host forces on fluid 0 (1 particle), 5, 15 and the emptied fluid 11: each is called once per step, the empty one with
    n = 0 and offsets {0}, and each one's additions land on its own rows only."""
    sc = S.scene_sixteen()
    assert len(sc["fluids"][0]["positions"]) == 1
    rig = Rig(sc, _maker(), [(0, 0), (5, 0), (15, 0), (S.SIXTEEN_EMPTIED, 0)])
    for _ in range(2):
        rig.step()
        empty = [cap for s, _, cap in rig.calls if s == S.SIXTEEN_EMPTIED]
        assert len(empty) == 1 and empty[0]["n"] == 0
        assert list(empty[0]["ff"]["offsets"]) == [0] and list(empty[0]["fb"]["offsets"]) == [0]
        assert len(empty[0]["boundaries"]) == 1 and len(empty[0]["boundaries"][0]["positions"]) == len(sc["boundaries"][0]["positions"])
    rig.finish("sixteen")


def test_host_force_ctx_with_lists_past_the_staging_rows():
    """The compressed block of test_gpu_neighbor_lists.py: lists longer than the 32 / 8 staging rows and the initial
    capacity of 64, which the search regrows."""
    r = S.R
    pts = scenes.jitter(scenes.block_lattice(13, 9, 11, r * 0.75), r, 23, amplitude=0.2)
    tank = scenes.open_tank((-r, -r, -r), (13 * 2 * r * 0.75 + r, 1.0, 11 * 2 * r * 0.75 + r), r)
    sc = dict(fluids=[dict(positions=pts, velocities=np.zeros_like(pts), density0=1000.0)], boundaries=[dict(positions=tank)])
    rig = Rig(sc, _maker(), [(0, 0)], pre=False)
    rig.step(dt=1e-5, iters=(1, 1))
    assert rig.w.stats()["max_neighbors"] > 64
    cap = rig.calls[0][2]
    assert (np.diff(cap["ff"]["offsets"]) > 32).mean() >= 0.25 and (np.diff(cap["fb"]["offsets"]) > 8).sum() >= 32
    rig.finish("compressed")


@pytest.mark.parametrize("edit", ["delete", "append", "refill_fluid_slot", "regrow_boundary_slot"])
def test_host_force_ctx_after_host_edits(edit):
    sc = S.scene_two_fluids()
    rig = Rig(sc, _maker(), [(0, 0), (1, 0)])
    rig.step()
    if edit == "delete":
        n = rig.w.num_particles(rig.fl[0]["h"])
        rig.delete(0, np.arange(n) % 5 == 2)
    elif edit == "append":
        rig.append(1, (sc["fluids"][1]["positions"][:40] + F(0.3) * np.array([0, 1, 0], F)).astype(F))
    elif edit == "refill_fluid_slot":
        rig.remove_fluid(1)
        f = dict(sc["fluids"][1], positions=(sc["fluids"][1]["positions"][::2] + F(0.01)).astype(F),
                 velocities=sc["fluids"][1]["velocities"][::2], density0=1200.0)
        assert rig.add_fluid(f) == 1
        rig.push_host(1, 0)
    elif edit == "regrow_boundary_slot":
        floor = sc["boundaries"][0]["positions"]
        bigger = np.concatenate([floor, floor[:200] + np.array([0, -2 * S.R, 0], F)]).astype(F)
        rig.remove_boundary(0)
        assert rig.add_boundary(dict(positions=bigger, velocities=np.zeros_like(bigger))) == 0
    for _ in range(2):
        rig.step()
    rig.finish("edit/" + edit)


def test_host_force_ctx_sees_this_steps_collider_particles():
    """A StaticSampling collider moved with set_collider_state between steps (boundary 1) and DynamicContactSampling of a
    Ball and a Cuboid just above the fluid (boundaries 2 and 3): the views and the boundary contacts are this step's
    particles.  The fluid is the sparse block (below rest density: it does not expand) and the shapes stay clear of it, so
    no particle is pushed and the positions are those read before."""
    sc = S.scene_gate()
    top = float(sc["fluids"][0]["positions"][:, 1].max())
    u = np.random.default_rng(3).normal(size=(300, 3))
    sphere = (0.12 * u / np.linalg.norm(u, axis=1)[:, None]).astype(F)
    rig = Rig(sc, _maker(), [(0, 0)], pre=False)
    for _ in range(3):
        rig.add_boundary(dict(positions=np.zeros((0, 3), F)))
    ws = (rig.w, rig.t)
    stat = [w.register_coupling(rig.bd[1][k], StaticSampling(sphere)) for w, k in zip(ws, ("h", "th"))]
    for w, k in zip(ws, ("h", "th")):
        ball = w.register_coupling(rig.bd[2][k], DynamicContactSampling(Ball(0.1)))
        box = w.register_coupling(rig.bd[3][k], DynamicContactSampling(Cuboid((0.1, 0.05, 0.1))))
        w.set_collider_state(ball, translation=(0.6, top + 0.17, 0.45))   # 0.07 above the fluid's top
        w.set_collider_state(box, translation=(0.25, top + 0.12, 0.6))     # 0.07 above it
    for p in ((0.3, top + 0.2, 0.3), (0.35, top + 0.19, 0.32), (0.42, top + 0.18, 0.35)):
        for w, c in zip(ws, stat):
            w.set_collider_state(c, translation=p, body=BODY_NONE)
        rig.step(gravity=S.ZERO_G)
        for b in (1, 2, 3):
            assert len(rig.w.read_boundary_particles(rig.bd[b]["h"])[0]) > 0, b
        assert (np.concatenate([cap["fb"]["j_model"] for _, _, cap in rig.calls]) == 1).any()
    rig.finish("colliders")


@pytest.mark.parametrize("flags", [(True, False), (False, True), (False, False)], ids=["contacts", "boundaries", "neither"])
def test_host_force_ctx_flags(flags):
    rig = Rig(S.scene_two_fluids(), _maker(), [(0, 0), (1, 0)], flags=flags)
    rig.step()
    rig.finish("flags/%d%d" % flags)


def test_host_forces_of_an_empty_fluid_are_called_once_per_step():
    """As predict_advection calls solve for every fluid (dfsph_solver.rs:580-603), a host force on a fluid whose particles
    were all deleted is called once per step, with n = 0 and offsets {0}; the legacy callback likewise with n = 0."""
    sc = S.scene_tail(33)
    sc["fluids"].append(dict(positions=np.zeros((0, 3), F), density0=900.0, deleted=sc["fluids"][0]["positions"][:5] + F(0.4)))
    w = LiquidWorld(DFSPHSolver(), particle_radius=S.R)
    fh, _ = S.populate(w, sc)
    seen = {"ctx": [], "legacy": []}

    def solve2(ctx):
        seen["ctx"].append((len(ctx.positions), list(ctx.fluid_fluid_contacts.offsets), list(ctx.fluid_boundaries_contacts.offsets),
                            len(ctx.boundaries), ctx.fluid_index))

    def solve(dt, inv_dt, h, pos, vel, dens, acc):
        seen["legacy"].append(len(pos))
        acc += 1.0   # nothing to add to

    w.push_host_force2(fh[1], solve2)
    w.push_host_force(fh[1], solve)
    for k in range(1, 3):
        w.step(S.DT, GRAVITY)
        assert seen["ctx"] == [(0, [0], [0], 1, fh[1] & 0xFFFF)] * k
        assert seen["legacy"] == [0] * k
    assert w.num_particles(fh[1]) == 0 and w.num_particles(fh[0]) == 33
    w.close()
