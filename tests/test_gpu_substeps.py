"""CFL-bounded substeps (sph_world_set_substepping, DESIGN.md section 12) on the device: off is off, a substepped step equals
the same substeps stepped by hand, the substep counts meet the float64 rule (oracle/ref64_substeps.py), snapshots continue
bit-identically, and the edges (refusals, steps that run no solver, the stats)."""
import math

import numpy as np
import pytest

from oracle import ref64_stages as S
from oracle import ref64_substeps as R64
from salva_b200 import BODY_DYNAMIC, DFSPHSolver, IISPHSolver, LiquidWorld, SphError, StaticSampling, scenes
from salva_b200.liquid_world import Ball, CouplingManager, DynamicContactSampling, Poly6Kernel, SpikyKernel

pytestmark = pytest.mark.gpu

F32 = np.float32
G = (0.0, -9.81, 0.0)
T = 1.0 / 60.0
STEPS = 3
K = {1: Poly6Kernel, 2: SpikyKernel}
LIBS = pytest.mark.parametrize("lib", ["cubic", "poly6+spiky"])
# (T, cfl, min, max): one substep; intermediate counts; the maximum binding.  The scenes' blocks start 2.4x over-dense and
# fly apart at up to a few hundred m/s after their first step, hence the wide range of cfl
REGIMES = dict(one=(S.DT, 50.0, 1, 10), mid=(S.DT, 1.0, 1, 64), max=(T, 0.01, 1, 4))
# force path -> (solver, scene, forces)
PATHS = dict(
    quiet=("dfsph", S.scene_block_forces, []),                                           # k_fold_integrate, no force
    xsph=("dfsph", S.scene_block, [scenes.xsph_viscosity(0.5, 0.0)]),                    # XSPH fused into the loop
    akinci=("dfsph", S.scene_block, [scenes.akinci2013_surface_tension(1.0, 0.0)]),      # Akinci fused into the loop
    two_fluids=("dfsph", S.scene_two_fluids, [scenes.xsph_viscosity(0.5, 0.0)]),          # separate force passes
    iisph_becker=("iisph", S.scene_block, [scenes.becker2009_elasticity(2.0e5, 0.3)]),
)


def _world(lib="cubic", solver="dfsph"):
    kd, kg = (0, 0) if lib == "cubic" else (1, 2)
    cls = DFSPHSolver if solver == "dfsph" else IISPHSolver
    return LiquidWorld(cls(K[kd], K[kg]) if kd else cls(), particle_radius=S.R, smoothing_factor=2.0)


def _make(path, lib):
    solver, scene, forces = PATHS[path]
    w = _world(lib, solver)
    fh, bh = S.populate(w, scene(), forces)
    return w, fh, bh, solver


def _obs(w, fh, solver):
    pv = [w.read_fluid(f) for f in fh]
    out = dict(P=np.concatenate([p for p, _ in pv]), V=np.concatenate([v for _, v in pv]),
               vc=np.concatenate([w.debug(f, "velocity_change") for f in fh]))
    if solver == "iisph":
        out["pressure"] = np.concatenate([w.debug(f, "pressure") for f in fh])
    return out


def _same(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k]), "%s: %s differs (max |d| = %g)" % (what, k, float(np.abs(a[k] - b[k]).max()))


def _velocities(w, fh):
    return np.concatenate([w.read_fluid(f)[1] for f in fh])


def _accelerations(w, fh):
    return np.concatenate([w.debug(f, "acceleration") for f in fh])


# ---- 1. off is off ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", sorted(PATHS))
@LIBS
def test_off_is_off(path, lib):
    """A world never configured and one set to max_substeps = 1 (which takes the split fold, the reduction and the separate
    integration on the quiet path) compute the same bits, step for step."""
    a, fa, _, solver = _make(path, lib)
    b, fb, _, _ = _make(path, lib)
    b.set_substepping(0.4, 1, 1)
    for k in range(STEPS):
        a.step(S.DT, G)
        b.step(S.DT, G)
        _same(_obs(a, fa, solver), _obs(b, fb, solver), "step %d" % k)
        sa, sb = a.stats(), b.stats()
        for key in ("n_divergence_iter", "n_pressure_iter", "n_divergence_eval", "n_pressure_eval", "n_substeps"):
            assert sa[key] == sb[key], key
        assert sa["n_substeps"] == 1 and list(a.substeps()) == [F32(S.DT)]


# ---- 2. + 3. a substepped step equals manual steps, and its counts meet the float64 rule --------------------------------------
def _pair(path, lib, regime):
    """World A substeps each step(T); world B steps every dt_k of A by hand.  Both stay bit-identical; A's stats are B's
    summed or last as specified; A's counts meet ref64_substeps.check on the v and a B saw (DFSPH: the velocities after
    the step, which the divergence loop folded in; IISPH: those before it)."""
    Tstep, cfl, mn, mx = REGIMES[regime]
    a, fa, _, solver = _make(path, lib)
    b, fb, _, _ = _make(path, lib)
    a.set_substepping(cfl, mn, mx)
    counts, near = [], 0
    for k in range(STEPS):
        a.step(Tstep, G)
        dts = a.substeps()
        sa = a.stats()
        assert sa["n_substeps"] == len(dts) >= 1
        per, states = [], []
        for dt in dts:
            v_before = _velocities(b, fb)
            b.step(float(dt), G)
            per.append(b.stats())
            states.append((v_before if solver == "iisph" else _velocities(b, fb), _accelerations(b, fb)))
        _same(_obs(a, fa, solver), _obs(b, fb, solver), "%s %s %s step %d" % (path, lib, regime, k))
        for key in ("n_divergence_iter", "n_pressure_iter", "n_divergence_eval", "n_pressure_eval"):
            assert sa[key] == sum(p[key] for p in per), key
        for key in ("last_divergence_error", "last_density_error", "n_contacts", "grid_dims", "n_fluid_particles"):
            assert sa[key] == per[-1][key], key
        assert sa["max_neighbors"] == max(p["max_neighbors"] for p in per)
        base = sum(p["kernel_launches"] for p in per) + len(dts)   # one k_cfl_max per substep
        if path == "quiet":
            assert sa["kernel_launches"] == base + len(dts)         # and the fused fold-and-integrate split in two
        elif path in ("xsph", "akinci"):
            assert base <= sa["kernel_launches"] <= base + len(dts)
        else:
            assert sa["kernel_launches"] == base
        res = R64.check(Tstep, dts, states, S.R, cfl, mn, mx)
        assert not res["failures"], res["failures"]
        near += len(res["near"])
        counts.append(len(dts))
    print("\nSUBSTEPS %s %s %s counts=%s near_integer=%d" % (path, lib, regime, counts, near))
    return counts


@pytest.mark.parametrize("regime", sorted(REGIMES))
@pytest.mark.parametrize("path", sorted(PATHS))
@LIBS
def test_a_substepped_step_equals_manual_steps(path, lib, regime):
    counts = _pair(path, lib, regime)
    _, _, mn, mx = REGIMES[regime]
    if regime == "one":
        assert counts == [1] * STEPS
    elif regime == "mid":
        assert any(1 < n < mx for n in counts), counts
    else:
        assert mx in counts, counts


@pytest.mark.parametrize("path", ["quiet", "xsph", "two_fluids", "iisph_becker"])
def test_a_substepped_step_equals_manual_steps_in_row_order(path, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    _pair(path, "cubic", "mid")


def _host_force_calls(path, regime):
    """(A's calls per step, B's calls per step) of a host force pushed on fluid 0."""
    Tstep, cfl, mn, mx = REGIMES[regime]
    out = []
    for substep in (True, False):
        w, fh, _, solver = _make(path, "cubic")
        calls = []

        def solve(dt, inv_dt, h, p, v, d, acc, calls=calls):
            calls.append((dt, inv_dt))
            acc += F32(0.25)   # the force reaches the state both worlds compare
        w.push_host_force(fh[0], solve)
        if substep:
            w.set_substepping(cfl, mn, mx)
        out.append((w, fh, calls, solver))
    return out


def test_host_force_calls_match_the_manual_steps():
    """A host NonPressureForce runs once per substep with that substep's lagging (dt, inv_dt), as B's steps see them."""
    (a, fa, ca, solver), (b, fb, cb, _) = _host_force_calls("two_fluids", "mid")
    Tstep = REGIMES["mid"][0]
    for k in range(STEPS):
        a.step(Tstep, G)
        dts = a.substeps()
        for dt in dts:
            b.step(float(dt), G)
        assert ca == cb
        _same(_obs(a, fa, solver), _obs(b, fb, solver), "host force step %d" % k)
    assert len(ca) > STEPS  # some step ran more than one substep


class _Recorder(CouplingManager):
    def __init__(self):
        self.calls, self.forces = [], []

    def update_boundaries(self, world, dt, inv_dt, h, particle_radius):
        self.calls.append(("update", dt, inv_dt))

    def transmit_forces(self, world, dt, inv_dt):
        self.calls.append(("transmit", dt, inv_dt))
        self.forces.append(world.read_boundary(world._test_b)[1].copy())


def test_coupling_manager_runs_once_per_substep():
    """update_boundaries and transmit_forces run per substep with the TimestepManager's values, and see the same boundary
    forces."""
    Tstep, cfl, mn, mx = REGIMES["mid"]
    ws = []
    for substep in (True, False):
        w, fh, bh, solver = _make("quiet", "cubic")
        w._test_b = bh[0]
        if substep:
            w.set_substepping(cfl, mn, mx)
        ws.append((w, fh, _Recorder()))
    (a, fa, ra), (b, fb, rb) = ws
    for k in range(STEPS):
        a.step_with_coupling(Tstep, G, ra)
        for dt in a.substeps():
            b.step_with_coupling(float(dt), G, rb)
        assert ra.calls == rb.calls
        for fa_, fb_ in zip(ra.forces, rb.forces):   # boundary forces are atomic sums: equal up to their order
            assert np.allclose(fa_, fb_, rtol=1e-4, atol=1e-5 * float(np.abs(fb_).max() + 1e-30))
        _same(_obs(a, fa, "dfsph"), _obs(b, fb, "dfsph"), "coupling step %d" % k)
    assert len(ra.calls) > 2 * STEPS


BOX = scenes.cuboid_surface((0.1, 0.08, 0.1), S.R).astype(F32)


def _collider_world(substep, cfl, mn, mx):
    w, fh, bh, _ = _make("quiet", "cubic")
    cs = w.register_coupling(w.add_boundary(np.zeros((0, 3), F32), want_forces=True), StaticSampling(BOX))
    cc = w.register_coupling(w.add_boundary(np.zeros((0, 3), F32)), DynamicContactSampling(Ball(0.1)))
    if substep:
        w.set_substepping(cfl, mn, mx)
    return w, fh, (cs, cc)


def _pose(w, cols, k):
    cs, cc = cols
    w.set_collider_state(cs, translation=(0.45, 0.3 - 0.01 * k, 0.4), body=BODY_DYNAMIC, linvel=(0.0, -0.6, 0.0),
                         angvel=(0.0, 0.5, 0.0), world_com=(0.45, 0.3 - 0.01 * k, 0.4))
    w.set_collider_state(cc, translation=(0.25, 0.55 - 0.02 * k, 0.3), body=BODY_DYNAMIC, linvel=(0.0, -1.2, 0.0),
                         world_com=(0.25, 0.55 - 0.02 * k, 0.3))


@pytest.mark.parametrize("regime", ["mid", "max"])
def test_colliders_sum_their_substep_impulses(regime):
    """StaticSampling and DynamicContactSampling colliders are posed from the same state every substep; A's impulse is the
    float32 left-to-right sum of B's per-step impulses, up to the order of the atomic reduction that forms each of them."""
    Tstep, cfl, mn, mx = REGIMES[regime]
    a, fa, ca = _collider_world(True, cfl, mn, mx)
    b, fb, cb = _collider_world(False, cfl, mn, mx)
    total = 0
    for k in range(STEPS):
        _pose(a, ca, k)
        a.step(Tstep, G)
        dts = a.substeps()
        seen = {c: [] for c in cb}
        for dt in dts:
            _pose(b, cb, k)
            b.step(float(dt), G)
            for c in cb:
                seen[c].append(b.collider_impulse(c))
        _same(_obs(a, fa, "dfsph"), _obs(b, fb, "dfsph"), "colliders step %d" % k)
        for x, y in zip(ca, cb):
            lin = ang = None
            for l_, g_ in seen[y]:
                lin = l_ if lin is None else (lin + l_).astype(F32)
                ang = g_ if ang is None else (ang + g_).astype(F32)
            la, ga = a.collider_impulse(x)
            # each impulse is a float atomicAdd reduction over the boundary, whose order varies from run to run: equal up to that
            for got, want in ((la, lin), (ga, ang)):
                assert np.allclose(got, want, rtol=1e-4, atol=1e-5 * float(np.abs(want).max() + 1e-30)), (k, got, want)
        total += len(dts)
    assert total > STEPS


def test_a_pending_delete_is_applied_once():
    """A delete issued before a substepped step is applied before its first substep, once."""
    Tstep, cfl, mn, mx = REGIMES["mid"]
    a, fa, _, solver = _make("xsph", "cubic")
    b, fb, _, _ = _make("xsph", "cubic")
    a.set_substepping(cfl, mn, mx)
    for w in (a, b):
        w.step(S.DT, G)
    n = a.num_particles(fa[0])
    mask = np.zeros(n, np.uint8)
    mask[::7] = 1
    a.delete_particles(fa[0], mask)
    b.delete_particles(fb[0], mask)
    a.step(Tstep, G)
    dts = a.substeps()
    assert len(dts) > 1
    for dt in dts:
        b.step(float(dt), G)
    assert a.num_particles(fa[0]) == n - int(mask.sum())
    _same(_obs(a, fa, solver), _obs(b, fb, solver), "after the delete")


# ---- 4. snapshots -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["xsph", "two_fluids", "iisph_becker"])
def test_snapshot_after_a_substepped_step_continues_bit_identically(path):
    Tstep, cfl, mn, mx = REGIMES["mid"]
    a, fa, _, solver = _make(path, "cubic")
    a.set_substepping(cfl, mn, mx)
    for _ in range(2):
        a.step(Tstep, G)
    blob = a.snapshot()
    b, fb, _, _ = _make(path, "cubic")
    b.set_substepping(cfl, mn, mx)
    b.restore(blob)
    for k in range(2):
        a.step(Tstep, G)
        b.step(Tstep, G)
        assert np.array_equal(a.substeps(), b.substeps())
        _same(_obs(a, fa, solver), _obs(b, fb, solver), "restored step %d" % k)


# ---- 5. edges ---------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing():
    w, fh, _, _ = _make("xsph", "cubic")
    w.set_substepping(math.inf, 3, 3)
    for args in ((math.nan, 1, 10), (-0.1, 1, 10), (-math.inf, 1, 10), (0.4, 0, 10), (0.4, 5, 4), (0.0, 0, 0)):
        with pytest.raises(SphError) as e:
            w.set_substepping(*args)
        assert e.value.status == 1, args
    w.step(S.DT, G)
    assert len(w.substeps()) == 3 and w.stats()["n_substeps"] == 3   # still (+inf, 3, 3)
    w.set_substepping(0.0, 1, 10)   # off
    w.step(S.DT, G)
    assert list(w.substeps()) == [F32(S.DT)]
    slab = LiquidWorld(particle_radius=S.R, slab_rank=0, slab_count=2)
    with pytest.raises(SphError) as e:
        slab.set_substepping(0.4, 1, 10)
    assert e.value.status == 1


@pytest.mark.parametrize("N", [2, 5])
def test_infinite_cfl_gives_n_equal_substeps(N):
    w, fh, _, _ = _make("quiet", "cubic")
    w.set_substepping(math.inf, N, N)
    w.step(T, G)
    dts = w.substeps()
    assert len(dts) == N and np.allclose(dts, T / N, rtol=4e-7, atol=0)
    assert abs(float(np.sum(dts.astype(np.float64))) - T) <= 2.0 ** -23 * T * N


def test_steps_that_run_no_solver():
    """dt <= FLT_EPSILON, and a world without fluid particles, behave as without substepping and report no substeps."""
    for substep in (False, True):
        w, fh, _, _ = _make("xsph", "cubic")
        if substep:
            w.set_substepping(0.1, 2, 10)
        p0 = w.read_fluid(fh[0])[0]
        for dt in (0.0, R64.FLT_EPS):
            w.step(dt, G)
            assert w.stats()["n_substeps"] == 0 and len(w.substeps()) == 0
        assert np.array_equal(w.read_fluid(fh[0])[0], p0)
        e = LiquidWorld(particle_radius=S.R)
        e.add_boundary(S.scene_block()["boundaries"][0]["positions"])
        if substep:
            e.set_substepping(0.1, 2, 10)
        e.step(T, G)
        assert e.stats()["n_substeps"] == 0 and len(e.substeps()) == 0
