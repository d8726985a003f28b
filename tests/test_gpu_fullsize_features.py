"""The step graph, CFL substeps, sources and sinks, and surface extraction at the benchmark's sizes, where their reductions,
scans and per-block logic run over thousands of blocks and past the scans' second level:
  1. sph_world_step_many against as many step() calls (tests/test_gpu_step_many.py's twin) at C2 in both grid orders and
     at C3, graph steps on the envelope (on_device == 1) and the step after the call; and a particle in the last slot of
     the sorted order that leaves the envelope mid-call;
  2. substepped steps against the same substeps stepped by hand (tests/test_gpu_substeps.py's twin) at C2, with the
     substep counts checked by oracle/ref64_substeps.py over every particle, and one isolated fast particle planted in
     the last slot (alone in the last warp), in slot 0 or in the middle: it alone makes the count >= 3;
  3. sinks and sources against the host-driven twin (tests/test_gpu_sources_sinks.py) at C2 (more than 2048 removals,
     box edges on particle coordinates, per-particle volumes), C5 (two IISPH fluids) and C3, whose N + 1 flags are scanned
     at three levels;
  4. the surface field against the float64 field (oracle/ref64_surface.py) on lattices past 2048^2 points, at C2 with its
     mesh and normals, and at C3.
Each test prints one FULLSIZE line: sizes, scan levels, counts, the worst err / bound and the device memory it used."""
import json
import time

import numpy as np
import pytest

import test_gpu_sources_sinks as SK
import test_gpu_step_many as SM
import test_gpu_substeps as SS
from oracle import ref64_stages as S
from oracle import ref64_substeps as R64
from oracle import ref64_surface as RS
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, scenes

pytestmark = pytest.mark.gpu

F = np.float32
G = scenes.GRAVITY
SCAN2 = S.SCAN_B * S.SCAN_B
ORDERS = {"h_order": "1", "row_order": "2"}
INF = np.inf


def _levels(n):
    """Levels of the block scan (scan_exclusive, scan_exclusive_k) over n entries of SCAN_B per block."""
    k = 1
    while n > S.SCAN_B:
        n = -(-n // S.SCAN_B)
        k += 1
    return k


class _Memory:
    """Device memory in use above what it was when the test began, sampled at the test's heavy points (mem_get_info:
    the whole device, so other work on it is counted too)."""

    def __init__(self):
        import torch
        self._info = torch.cuda.mem_get_info
        self.base = self.used()
        self.peak = 0.0

    def used(self):
        free, total = self._info()
        return (total - free) / float(1 << 30)

    def sample(self):
        self.peak = max(self.peak, self.used() - self.base)

    def gb(self):
        return round(self.peak, 2)


def _report(kind, **tags):
    print("\nFULLSIZE %s" % json.dumps(dict(test=kind, **tags)))


def _scene(base, seed):
    """A bench scene with its forces, seeded random velocities (sigma 0.2 m/s) and still boundaries."""
    rng = np.random.default_rng(seed)
    fl = [dict(f, velocities=rng.normal(0, 0.2, f["positions"].shape).astype(F)) for f in base["fluids"]]
    bd = [dict(positions=b["positions"], velocities=np.zeros_like(b["positions"])) for b in base["boundaries"]]
    return dict(base, fluids=fl, boundaries=bd)


def _plant(sc, p, v):
    """Appends one particle (position p, velocity v) to fluid 0: it is the last in caller order."""
    f = sc["fluids"][0]
    sc["fluids"][0] = dict(f, positions=np.concatenate([f["positions"], np.asarray([p], F)]).astype(F),
                           velocities=np.concatenate([f["velocities"], np.asarray([v], F)]).astype(F))
    return sc


def _table_index(sc, xysub):
    P = np.concatenate([f["positions"] for f in sc["fluids"]])
    B = np.concatenate([b["positions"] for b in sc["boundaries"]])
    h = F(F(sc["particle_radius"]) * F(2.0) * F(2.0))
    return S.cell_table(P, B, h, xysub)[0]


def _twins(sc, solver=DFSPHSolver):
    out = []
    for _ in range(2):
        w = LiquidWorld(solver(), particle_radius=sc["particle_radius"], smoothing_factor=2.0)
        fh, bh = scenes.populate(w, sc)
        out.append((w, fh, bh))
    return out


def _close(pair):
    for w, _, _ in pair:
        w.close()


# ---- 1. step_many against step() -------------------------------------------------------------------------------------------
def _one_more_step(pair, dt):
    """One step() on both: the graph world's grid starts from the bounds its last graph step reduced."""
    (w1, f1, b1), (w2, f2, b2) = pair
    for w in (w1, w2):
        w.step(dt, G)
    SM._same(SM._obs(w1, f1, b1), SM._obs(w2, f2, b2), "the step after step_many")
    assert w1.step_records() == w2.step_records()


def _step_many_case(sc, K, label, **tags):
    t0 = time.time()
    mem = _Memory()
    n = sum(len(f["positions"]) for f in sc["fluids"])
    pair = _twins(sc)
    try:
        rec = SM._drive(pair, K, sc["dt"], G)
        mem.sample()
        on = [r["on_device"] for r in rec]
        assert on == [0] + [1] * (K - 1), on   # steps 2..K ran in the graph, on the envelope
        _one_more_step(pair, sc["dt"])
        _report("step_many", scene=label, n=n, K=K, on_device=on, pass_blocks=-(-n // S.PASS_T),
                evals=[(r["n_divergence_eval"], r["n_pressure_eval"]) for r in rec], max_neighbors=rec[-1]["max_neighbors"],
                device_gb=mem.gb(), seconds=round(time.time() - t0), **tags)
    finally:
        _close(pair)


@pytest.mark.parametrize("order", sorted(ORDERS))
def test_c2_step_many_equals_steps(order, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", ORDERS[order])   # read when the world is created
    _step_many_case(_scene(scenes.scene_c2(compress=0.93), 0xC2), 8, "c2", order=order)


def test_c3_step_many_equals_steps():
    sc = _scene(scenes.scene_c3(compress=0.93), 0xC3)
    assert len(sc["fluids"][0]["positions"]) == 10_077_696
    _step_many_case(sc, 4, "c3", order="h_order")


def test_c2_step_many_leaves_the_envelope():
    """A particle 0.25 m above the fluid in its highest x cell holds the last table index: the last slot of the sorted
    order, alone in the last warp and block (N = 10^6 + 1).  At 300 m/s upwards it is inside the envelope of step 1's
    bounds (fluid and tank, 4 cells of margin) after steps 1 and 2 and past it after step 3 (with no neighbour after step
    1, it flies at 300 m/s less gravity).  The graph must see it leave, stop, and the call must finish on the host path,
    equal to the twin."""
    t0 = time.time()
    mem = _Memory()
    sc = _scene(scenes.scene_c2(compress=0.93), 0xC2)
    P = sc["fluids"][0]["positions"]
    top = P[np.argmax(P[:, 0])]
    _plant(sc, (top[0], 4.9, 2.3), (0.0, 300.0, 0.0))
    n = len(P) + 1
    idx = _table_index(sc, 1)
    assert int(np.argmax(idx)) == n - 1 and int((idx == idx.max()).sum()) == 1 and n % 32 == 1
    dt, K = sc["dt"], 6
    pair = _twins(sc)
    try:
        (w1, f1, b1), (w2, f2, b2) = pair
        assert w1.step_many(dt, K, gravity=G) == K
        rec1 = w1.step_records()
        rec2, left = [], None
        h = w2.h
        blo, bhi = SM._cells(sc["boundaries"][0]["positions"], h)
        for k in range(K):
            w2.step(dt, G)
            rec2 += w2.step_records()
            lo, hi = SM._cells(w2.read_fluid(f2[0])[0], h)
            if k == 0:
                env_lo, env_hi = np.minimum(lo, blo) - 4, np.maximum(hi, bhi) + 4
            elif left is None and ((lo < env_lo).any() or (hi > env_hi).any()):
                left = k
        mem.sample()
        SM._same(SM._obs(w1, f1, b1), SM._obs(w2, f2, b2), "step_many leaving the envelope")
        assert SM._strip(rec1) == SM._strip(rec2)
        on = [r["on_device"] for r in rec1]
        assert left in (2, 3), left
        # the graph ran up to the step that left, and the next step ran on the per-step path
        assert on[:left + 1] == [0] + [1] * left and on[left + 1] == 0, (left, on)
        _one_more_step(pair, dt)
        _report("step_many_envelope_exit", scene="c2", n=n, K=K, left_at_step=left + 1, on_device=on,
                device_gb=mem.gb(), seconds=round(time.time() - t0))
    finally:
        _close(pair)


# ---- 2. CFL substeps --------------------------------------------------------------------------------------------------------
# cfl, min, max.  R / d = T |v + a R| / (2 r cfl): at T = 1 ms and r = 0.025 the field's few m/s give well under 1 (one
# substep) and the outlier's 160 m/s gives 3.2, 2.4, 1.6, 0.8 over its substeps (4 substeps, no ratio near an integer)
CFL = (1.0, 1, 10)
OUTLIER = 160.0


def _outlier_scene(where):
    """C2 with one isolated particle (more than h from any other, fluid or boundary) flying away at OUTLIER m/s: beyond the
    fluid's highest x cell (the last table index: the last slot, alone in the last warp), beyond its lowest (slot 0, past
    the tank wall), or above the middle of its top."""
    sc = _scene(scenes.scene_c2(compress=0.93), 0xC2)
    P = sc["fluids"][0]["positions"]
    lo, hi = P.min(0), P.max(0)
    mid = (lo + hi) / 2
    p, v = dict(last=((hi[0] + 0.3, mid[1], mid[2]), (OUTLIER, 0.0, 0.0)),
                first=((lo[0] - 0.3, mid[1], mid[2]), (-OUTLIER, 0.0, 0.0)),
                middle=((mid[0], hi[1] + 0.3, mid[2]), (0.0, OUTLIER, 0.0)))[where]
    return _plant(sc, p, v)


@pytest.mark.parametrize("where,order", [("last", "h_order"), ("first", "h_order"), ("middle", "h_order"),
                                         ("last", "row_order")])
def test_c2_substeps_with_an_outlier(where, order, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", ORDERS[order])
    t0 = time.time()
    mem = _Memory()
    sc = _outlier_scene(where)
    n = sum(len(f["positions"]) for f in sc["fluids"])
    idx = _table_index(sc, int(ORDERS[order]))
    rank = int((idx < idx[-1]).sum())   # the outlier's slot in the sorted order (alone in its cell)
    assert int((idx == idx[-1]).sum()) == 1
    assert {"last": rank == n - 1, "first": rank == 0, "middle": n // 4 < rank < 3 * n // 4}[where], (where, rank)
    cfl, mn, mx = CFL
    r, T = sc["particle_radius"], sc["dt"]
    pair = _twins(sc)
    try:
        (a, fa, _), (b, fb, _) = pair
        a.set_substepping(cfl, mn, mx)
        counts, field, near = [], [], 0
        for k in range(2):
            a.step(T, G)
            dts = a.substeps()
            sa = a.stats()
            assert sa["n_substeps"] == len(dts)
            per, states = [], []
            for dt in dts:
                b.step(float(dt), G)
                per.append(b.stats())
                states.append((SS._velocities(b, fb), SS._accelerations(b, fb)))
            mem.sample()
            SS._same(SS._obs(a, fa, "dfsph"), SS._obs(b, fb, "dfsph"), "%s %s step %d" % (where, order, k))
            for key in ("n_divergence_iter", "n_pressure_iter", "n_divergence_eval", "n_pressure_eval"):
                assert sa[key] == sum(p[key] for p in per), key
            for key in ("last_divergence_error", "last_density_error", "n_contacts", "grid_dims", "n_fluid_particles"):
                assert sa[key] == per[-1][key], key
            res = R64.check(T, dts, states, r, cfl, mn, mx)   # every particle, every substep
            assert not res["failures"], res["failures"]
            near += len(res["near"])
            v, acc = states[0]
            field.append(R64.choose(v[:-1], acc[:-1], T, r, cfl, mn, mx, 0)[0])   # without the outlier
            counts.append(len(dts))
        assert field == [1, 1], field
        assert all(c >= 3 for c in counts), counts
        _report("substeps", scene="c2", where=where, order=order, n=n, slot=rank, counts=counts, without_outlier=field,
                near_integer=near, device_gb=mem.gb(), seconds=round(time.time() - t0))
    finally:
        _close(pair)


# ---- 3. sources and sinks ---------------------------------------------------------------------------------------------------
def _edit_scene(base, seed, solver, sinks=(), sources=(), volumes=None):
    """The twin's scene (tests/test_gpu_sources_sinks.py scene()) from a bench scene."""
    sc = _scene(base, seed)
    fl = [dict(positions=f["positions"], velocities=f["velocities"], density0=f["density0"], forces=f["forces"])
          for f in sc["fluids"]]
    if volumes is not None:
        fl[0]["volumes"] = volumes
    return dict(solver=solver, particle_radius=sc["particle_radius"], dt=sc["dt"], fluids=fl,
                boundaries=[b["positions"] for b in sc["boundaries"]], sinks=list(sinks), sources=list(sources),
                forces_wanted=False)


def _sheet(n, r, origin, vy):
    """n x n template particles at spacing 2r in the plane y = origin[1]."""
    g = np.arange(n, dtype=F) * F(2 * r)
    p = np.stack(np.meshgrid(g + F(origin[0]), np.array([origin[1]], F), g + F(origin[2]), indexing="ij"), -1)
    p = p.reshape(-1, 3).astype(F)
    v = np.zeros_like(p)
    v[:, 1] = vy
    return p, v


def _drain(fi, y):
    return (fi, (-INF, -INF, -INF), (INF, y, INF), 0)


def _run_edits(sc, steps, label, check=None, **tags):
    t0 = time.time()
    mem = _Memory()
    P = SK.Pair(sc)
    try:
        per = []
        for k in range(steps):
            n0 = P.a.stats()["n_fluid_particles"] if k else sum(len(f["positions"]) for f in sc["fluids"])
            want = P.step(sc["dt"])   # asserts step_edits against the twin's numpy box counts
            mem.sample()
            per.append(dict(n0=n0, scan_levels=_levels(n0 + 1), edits=[list(w) for w in want]))
            if check:
                check(P, k)
        _report("sources_sinks", scene=label, steps=per, device_gb=mem.gb(), seconds=round(time.time() - t0), **tags)
        return per
    finally:
        for w in (P.a, P.b):
            w.close()


def _exact_box(P, lattice_n, a, b):
    """A box whose lo is particle a's position and whose hi is particle b's (lattice indices (i, j, k))."""
    ia = (a[0] * lattice_n + a[1]) * lattice_n + a[2]
    ib = (b[0] * lattice_n + b[1]) * lattice_n + b[2]
    lo, hi = P[ia], P[ib]
    assert np.all(lo < hi)
    return ia, ib, (0, lo, hi, 0)


@pytest.mark.parametrize("volumes", [False, True], ids=["default_volumes", "volumes"])
def test_c2_sources_and_sinks(volumes):
    """A drain under the lowest lattice layer (10 000 removals in the first step, spread over every x cell), a box from one
    particle's coordinates to another's (the first removed, the second kept), and a 10 x 10 source firing every step; with
    per-particle volumes the host compacts its volume column by the list of more than 2048 removed indices."""
    base = scenes.scene_c2(compress=0.93)
    r = base["particle_radius"]
    P = base["fluids"][0]["positions"]
    ia, ib, box = _exact_box(P, 100, (50, 50, 50), (52, 52, 52))
    src = _sheet(10, r, (2.0, 4.9, 2.0), -5.0)   # 0.27 m above the fluid; 5 mm between firings
    vol = None
    if volumes:
        vol = (r ** 3 * 6.4 * np.random.default_rng(5).uniform(0.95, 1.05, len(P))).astype(F)
    sc = _edit_scene(base, 0xC2, DFSPHSolver(), sinks=[_drain(0, 0.05), box], sources=[(0, src[0], src[1], 1)], volumes=vol)

    def check(pair, k):
        if k == 0:
            ids = pair.a.read_ids(pair.fa[0])
            assert ia not in ids and ib in ids   # lo <= x removes, x < hi keeps

    per = _run_edits(sc, 4, "c2", check=check, volumes=volumes)
    assert per[0]["edits"][0][0] > 2048 and per[0]["scan_levels"] == 2
    assert all(p["edits"][0][1] == 100 for p in per)


def test_c5_sources_and_sinks():
    """Two IISPH fluids with Becker2009: a source into fluid 0 every step (fluid 1's original indices move up), sink boxes
    holding exactly the last particle of fluid 0 and the first of fluid 1, and a domain sink."""
    base = scenes.scene_c5()
    r = base["particle_radius"]
    last0 = base["fluids"][0]["positions"][-1]
    first1 = base["fluids"][1]["positions"][0]
    one = lambda fi, p: (fi, p, np.nextafter(p, F(INF)), 0)   # a box that holds exactly p
    src = _sheet(10, r, (6.0, 1.0, 2.0), -5.0)   # beside both blocks
    sinks = [one(0, last0), one(1, first1), (1, (-1.0, -1.0, -1.0), (11.0, 12.0, 6.0), 1)]
    sc = _edit_scene(base, 0xC5, IISPHSolver(), sinks=sinks, sources=[(0, src[0], src[1], 1)])
    n0 = len(base["fluids"][0]["positions"])

    def check(pair, k):
        if k == 0:
            assert n0 - 1 not in pair.a.read_ids(pair.fa[0]) and 0 not in pair.a.read_ids(pair.fa[1])

    per = _run_edits(sc, 3, "c5", check=check)
    assert per[0]["edits"] == [[1, 100], [1, 0]], per[0]
    assert all(p["edits"][0][1] == 100 for p in per)


def test_c3_sources_and_sinks():
    """C3's N + 1 > 2048^2 flags: the K = 2 scan of the keep and removed flags recurses to its third level."""
    base = scenes.scene_c3(compress=0.93)
    r = base["particle_radius"]
    src = _sheet(10, r, (4.0, 10.5, 4.0), -5.0)   # 0.48 m above the fluid
    sc = _edit_scene(base, 0xC3, DFSPHSolver(), sinks=[_drain(0, 0.05)], sources=[(0, src[0], src[1], 1)])
    per = _run_edits(sc, 3, "c3")
    assert per[0]["n0"] + 1 > SCAN2 and all(p["scan_levels"] == 3 for p in per)
    assert per[0]["edits"][0][0] > 2048


# ---- 4. surface extraction --------------------------------------------------------------------------------------------------
def _field_sample(dims, n_random, seed):
    """Lattice point indices (x fastest): n_random seeded random ones, every point of the first and last x planes, the
    first and last 2048 points (the first and last blocks of the field pass and of the count scan), and every point whose
    index is within 2 of a multiple of 2048 or 2048^2 (the count scan's block and level seams)."""
    npts = int(np.prod(dims, dtype=np.int64))
    p = np.arange(npts, dtype=np.int64)
    keep = (p % dims[0] == 0) | (p % dims[0] == dims[0] - 1) | (p < S.SCAN_B) | (p >= npts - S.SCAN_B)
    for m in (S.SCAN_B, SCAN2):
        q = p % m
        keep |= (q <= 2) | (q >= m - 2)
    rand = np.random.default_rng(seed).choice(npts, size=min(n_random, npts), replace=False)
    return np.union1d(np.nonzero(keep)[0], rand)


def _field_check(w, fluids, vol, label, mem, t0, mesh=False):
    phi, o, s = w.surface_field()
    dims = np.array(phi.shape[::-1], np.int64)
    npts = int(np.prod(dims))
    assert npts + 1 > SCAN2, npts   # the vertex-count scan runs at level 2 and beyond
    sel = _field_sample(dims, 200_000, 11)
    cx, cy, cz = RS.coords(o, dims, s)
    pts = np.stack([cx[sel % dims[0]], cy[(sel // dims[0]) % dims[1]], cz[sel // (dims[0] * dims[1])]], 1)
    pos = np.concatenate([w.read_fluid(f)[0] for f in fluids])
    h = float(w.h)
    ref, bound = RS.field64(pos, vol, pts, h)
    err = np.abs(phi.reshape(-1)[sel].astype(np.float64) - ref)
    ratio = err / np.maximum(bound, 1e-300)
    assert np.all(err <= bound), "phi off by %g > bound at %d points" % (float(err.max()), int((err > bound).sum()))
    assert phi.max() > 0.6 and (ref > 0).sum() > len(sel) // 10
    tags = dict(scene=label, lattice=dims.tolist(), npts=npts, count_scan_levels=_levels(npts + 1), sample=len(sel),
                worst_field=round(float(ratio.max()), 5))
    if mesh:
        v, t, nrm = w.read_surface(normals=True)
        t1 = time.time()
        rv, rt = RS.polygonise(phi, o, dims, s, 0.6)
        tags["polygonise_seconds"] = round(time.time() - t1)
        assert len(t) > 1000
        assert np.array_equal(rt, t)
        assert np.array_equal(rv.view(np.uint32), v.view(np.uint32))
        pick = np.random.default_rng(12).choice(len(v), size=min(100_000, len(v)), replace=False)
        n64, m, gb = RS.normals64(pos, vol, v[pick], h)
        ok = m > 1000.0 * gb
        assert ok.mean() > 0.9
        dev = np.linalg.norm(nrm[pick].astype(np.float64) - n64, axis=1)
        allowed = 2.0 * np.sqrt(3.0) * gb / np.where(ok, m, 1.0) + 1e-5
        assert np.all(dev[ok] <= allowed[ok]), float(dev[ok].max())
        tags.update(vertices=len(v), triangles=len(t), normals_sample=int(ok.sum()),
                    worst_normal=round(float((dev[ok] / allowed[ok]).max()), 5))
    _report("surface", device_gb=mem.gb(), seconds=round(time.time() - t0), **tags)


def _default_volume(r):
    """The engine's default particle volume r^3 * 6.4, in its float32 operation order."""
    r = F(r)
    return F(r * r * r * F(6.4))


@pytest.mark.parametrize("scene", ["c2", "c3"])
def test_surface_field_past_2048_squared_points(scene):
    """C2 after 5 steps (its mesh too: the float32 restatement of the GPU field's polygonisation, and the normals) and C3
    after one, at lattice spacing r over the default box.  The default box is the fluid grown by h, so the lattice's last
    points have no contact; C3 is sampled a second time on a box whose hi corner lies 2 m inside the fluid, so that the
    last block of the field pass holds points with contacts."""
    t0 = time.time()
    mem = _Memory()
    base = scenes.scene_c2(compress=0.93) if scene == "c2" else scenes.scene_c3(compress=0.93)
    sc = _scene(base, 0x5F)
    r = sc["particle_radius"]
    w = LiquidWorld(DFSPHSolver(), particle_radius=r, smoothing_factor=2.0)
    try:
        fh, _ = scenes.populate(w, sc)
        for _ in range(5 if scene == "c2" else 1):
            w.step(sc["dt"], G)
        w.extract_surface(iso=0.6, spacing=r, normals=scene == "c2")
        mem.sample()
        _field_check(w, fh, _default_volume(r), scene, mem, t0, mesh=scene == "c2")
        if scene == "c3":
            w.extract_surface(iso=0.6, spacing=r, box=((-0.2, -0.2, -0.2), (8.0, 8.0, 8.0)), normals=False)
            mem.sample()
            phi = w.surface_field()[0]
            assert phi.reshape(-1)[-1] > 0.6   # the last lattice point is inside the fluid
            _field_check(w, fh, _default_volume(r), "c3_clipped", mem, t0)
    finally:
        w.close()
