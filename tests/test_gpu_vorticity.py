"""Vorticity confinement on the device (include/sph.h SPH_FORCE_VORTICITY_CONFINEMENT, DESIGN.md section 18): each pass per
particle against the float64 reference (oracle/ref64_vorticity.py), the rigid-rotation closed form, step_many
against K steps, determinism, snapshots, isolation from the other fluids, the selectors and refusals, the device memory, and
what the force does to a rotating blob."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref64  # noqa: E402
from oracle import ref64_stages as S  # noqa: E402
from oracle import ref64_vorticity as RV  # noqa: E402
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, SphError, VorticityConfinement, scenes  # noqa: E402
from salva_b200.liquid_world import Poly6Kernel, SpikyKernel  # noqa: E402

F = np.float32
G = (0.0, -9.81, 0.0)
EPS = 0.05
LIBS = dict(cubic=(0, 0), poly6_spiky=(1, 2))
K = {1: Poly6Kernel, 2: SpikyKernel}


def _make(kd=0, kg=0, solver="dfsph"):
    cls = DFSPHSolver if solver == "dfsph" else IISPHSolver

    def make(**kw):
        s = cls(K[kd], K[kg]) if kd else cls()
        for k, v in kw.items():
            setattr(s, k, v)
        return LiquidWorld(s, particle_radius=S.R, smoothing_factor=2.0)
    return make


def _report(c, name, kd, kg, solver):
    print("\nREF64 %s" % json.dumps(dict(scene=name, force="vorticity", solver=solver, kernels=[kd, kg],
                                         worst={k: round(v, 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v})))
    assert not c.flagged(), c.worst


# ---- each pass against the float64 reference ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(S.SCENES))
@pytest.mark.parametrize("lib", sorted(LIBS))
def test_every_vorticity_pass_meets_its_bound(name, lib):
    kd, kg = LIBS[lib]
    c = RV.Checks(_make(kd, kg), S.SCENES[name](), kw=kd, kg=kg)
    c.vorticity(EPS)
    _report(c, name, kd, kg, "dfsph")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["block", "pairs", "two_fluids", "far"])
def test_every_vorticity_pass_meets_its_bound_in_row_order(name, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    c = RV.Checks(_make(), S.SCENES[name]())
    c.vorticity(EPS)
    _report(c, name, 0, 0, "dfsph")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(S.SCENES))
@pytest.mark.parametrize("lib", sorted(LIBS))
def test_every_vorticity_pass_meets_its_bound_under_iisph(name, lib):
    kd, kg = LIBS[lib]
    c = RV.Checks(_make(kd, kg, "iisph"), S.SCENES[name](), kw=kd, kg=kg)
    c.vorticity(EPS, iisph=True)
    _report(c, name, kd, kg, "iisph")


@pytest.mark.gpu
@pytest.mark.parametrize("lib", sorted(LIBS))
def test_rigid_rotation_on_the_device_gives_twice_kappa_omega(lib):
    """A full cubic lattice at rest spacing rotating rigidly: at interior particles omega = 2 kappa Omega, kappa from the
    lattice and the step's densities in float64."""
    kd, kg = LIBS[lib]
    n = 11
    a = (np.arange(n) - n // 2) * (2 * S.R)
    P = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3).astype(F)
    Om = np.array([0.4, -1.1, 0.7])
    V = np.cross(Om, P.astype(np.float64)).astype(F)
    w = _make(kd, kg)()
    fh = w.add_fluid(P, velocities=V)
    w.push_force(fh, *scenes.vorticity_confinement(EPS))
    w.force_iterations(0, 0)
    w.step(S.DT, S.ZERO_G)
    om, dens = w.debug(fh, "vorticity").astype(np.float64), w.debug(fh, "density").astype(np.float64)
    ps = ref64.Passes(S.kernel_h(F(S.R), 2.0), P, np.zeros(len(P), int), np.full(len(P), F(1000.0), F),
                      np.full(len(P), F(S.R) ** 3 * F(8.0 * 0.8) * F(1000.0), F), np.zeros((0, 3), F), np.zeros(0, int), kg=kg)
    g, _, _ = ps._g(ps.ff)
    kappa = np.bincount(ps.ff.i, ps.mass[ps.ff.j] / dens[ps.ff.j] * np.abs(g) * ps.ff.d2, len(P)) / 3.0
    inside = np.abs(P.astype(np.float64)).max(1) + ps.h <= a.max() + 1e-6
    assert inside.sum() >= 27
    want = 2 * kappa[inside, None] * Om
    err = np.abs(om[inside] - want).max() / np.abs(want).max()
    print("rigid rotation (%s): kappa %.6f..%.6f, max relative error %.2e" % (lib, kappa[inside].min(), kappa[inside].max(), err))
    assert err < 1e-4


# ---- step_many, determinism, snapshots -----------------------------------------------------------------------------------------
ORDERS = dict(alone=[scenes.vorticity_confinement(EPS)],
              after_xsph_akinci=[scenes.xsph_viscosity(0.5, 0.0), scenes.akinci2013_surface_tension(1.0, 0.0), scenes.vorticity_confinement(EPS)],
              first=[scenes.vorticity_confinement(EPS), scenes.xsph_viscosity(0.5, 0.0), scenes.akinci2013_surface_tension(1.0, 0.0)])


def _world(forces, lib="cubic", scene=S.scene_block):
    w = _make(*LIBS[lib])()
    fh, bh = S.populate(w, scene(), forces)
    return w, fh, bh


def _obs(w, fh, bh):
    o = {}
    for k, f in enumerate(fh):
        o["P%d" % k], o["V%d" % k] = w.read_fluid(f)
        for sel in ("velocity_change", "acceleration", "vorticity", "vorticity_eta"):
            o["%s%d" % (sel, k)] = w.debug(f, sel)
    return o


def _same(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), "%s: %s differs (max |d| = %g)" % (what, k, float(np.abs(a[k] - b[k]).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("order", sorted(ORDERS))
@pytest.mark.parametrize("lib", sorted(LIBS))
def test_step_many_equals_steps(order, lib):
    Kn = 8
    w1, f1, b1 = _world(ORDERS[order], lib)
    w2, f2, b2 = _world(ORDERS[order], lib)
    assert w1.step_many(S.DT, Kn, gravity=G) == Kn
    rec = w1.step_records()
    for _ in range(Kn):
        w2.step(S.DT, G)
    _same(_obs(w1, f1, b1), _obs(w2, f2, b2), "step_many(%d) %s" % (Kn, order))
    # step 1 runs per step, step 2 in the graph (later steps fall back to the per-step path once the block leaves the envelope)
    assert rec[0]["on_device"] == 0 and rec[1]["on_device"] == 1, [r["on_device"] for r in rec]


@pytest.mark.gpu
def test_runs_are_deterministic():
    obs = []
    for _ in range(2):
        w, fh, bh = _world(ORDERS["after_xsph_akinci"])
        for _ in range(6):
            w.step(S.DT, G)
        obs.append(_obs(w, fh, bh))
    _same(obs[0], obs[1], "run to run")


@pytest.mark.gpu
def test_snapshot_then_continuation_is_bit_identical():
    a, fa, ba = _world(ORDERS["alone"])
    for _ in range(4):
        a.step(S.DT, G)
    blob = a.snapshot()
    for _ in range(4):
        a.step(S.DT, G)
    b, fb, bb = _world(ORDERS["alone"])
    b.restore(blob)
    for _ in range(4):
        b.step(S.DT, G)
    _same(_obs(a, fa, ba), _obs(b, fb, bb), "snapshot")


@pytest.mark.gpu
def test_the_other_fluid_is_untouched():
    """Vorticity confinement on fluid 1 only: fluid 0's accelerations are those of a world without it, bit for bit."""
    outs = []
    for with_vc in (False, True):
        w = _make()()
        sc = S.scene_two_fluids()
        fh, bh = S.populate(w, sc)
        w.push_force(fh[0], *scenes.xsph_viscosity(0.5, 0.0))
        if with_vc:
            w.push_force(fh[1], *scenes.vorticity_confinement(EPS))
        w.step(S.DT, G)
        outs.append((w.debug(fh[0], "acceleration"), w.debug(fh[1], "acceleration")))
    assert np.array_equal(outs[0][0], outs[1][0])
    assert not np.array_equal(outs[0][1], outs[1][1])


# ---- selectors and refusals ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_selectors_are_refused_before_a_solve_and_after_an_append_and_have_width_three():
    w, fh, bh = _world(ORDERS["alone"], scene=lambda: S.scene_tail(33))
    for sel in ("vorticity", "vorticity_eta"):
        with pytest.raises(SphError):
            w.debug(fh[0], sel)
    w.step(S.DT, G)
    for sel in ("vorticity", "vorticity_eta"):
        assert w.debug(fh[0], sel).shape == (33, 3)
    w.append_particles(fh[0], np.array([[0.9, 0.9, 0.9]], F))
    for sel in ("vorticity", "vorticity_eta"):
        with pytest.raises(SphError):
            w.debug(fh[0], sel)
    w.step(S.DT, G)
    assert w.debug(fh[0], "vorticity").shape == (34, 3)
    # a fluid without the force: refused, as He2014's selectors are
    w2, fh2, _ = _world([scenes.xsph_viscosity(0.5, 0.0)], scene=lambda: S.scene_tail(33))
    w2.step(S.DT, G)
    with pytest.raises(SphError):
        w2.debug(fh2[0], "vorticity")


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [0.0, -1.0, float("nan"), float("inf"), float("-inf")])
def test_a_bad_eps_is_refused_and_changes_nothing(eps):
    ref, fr, br = _world(ORDERS["alone"])
    w, fh, bh = _world(ORDERS["alone"])
    with pytest.raises(SphError):
        w.push_force(fh[0], *scenes.vorticity_confinement(eps))
    with pytest.raises(SphError):
        w.push_force(fh[0], VorticityConfinement.kind, VorticityConfinement(eps).params)
    for x in (ref, w):
        for _ in range(3):
            x.step(S.DT, G)
    _same(_obs(ref, fr, br), _obs(w, fh, bh), "after a refused push")


@pytest.mark.gpu
def test_slab_worlds_are_refused():
    import ctypes as C

    from salva_b200 import _lib
    L = _lib.lib()
    d = _lib.WorldDesc()
    L.sph_world_desc_default(C.byref(d))
    d.particle_radius = S.R
    d.slab_count = 2
    d.slab_rank = 0
    w = C.c_void_p()
    if L.sph_world_create(C.byref(d), C.byref(w)) != 0:
        pytest.skip("this build refuses a slab world at creation")
    try:
        pts = S.scene_tail(31)["fluids"][0]["positions"]
        h = C.c_uint32()
        assert L.sph_fluid_add(w, pts.ctypes.data_as(C.POINTER(C.c_float)), None, None, len(pts), C.c_float(1000.0), 1, 0xFFFFFFFF,
                               C.byref(h)) == 0
        f = _lib.ForceDesc()
        f.kind = scenes.VORTICITY
        f.p[0] = EPS
        assert L.sph_fluid_push_force(w, h.value, C.byref(f)) == 1
    finally:
        L.sph_world_destroy(w)


# ---- device memory ------------------------------------------------------------------------------------------------------------
def _lifetime_child():
    import torch
    free = []
    pts = scenes.block_lattice(320, 3, 320, S.R)  # 307 200 particles: 9.4 MiB of vorticity scratch
    for _ in range(1 + 6):
        w = LiquidWorld(particle_radius=S.R)
        fh = w.add_fluid(pts)
        w.push_force(fh, *scenes.vorticity_confinement(EPS))
        w.step(S.DT, S.ZERO_G)
        w.close()
        free.append(torch.cuda.mem_get_info()[0])
    print("LIFETIME " + json.dumps({"free": free}))


@pytest.mark.gpu
def test_destroyed_world_returns_the_vorticity_scratch():
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "lifetime"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("LIFETIME ")][-1]
    free = np.asarray(json.loads(line[len("LIFETIME "):])["free"], np.float64)
    drops = -np.diff(free) / float(1 << 20)
    print("vorticity lifetime: median drop %.2f MiB per cycle, drops %s" % (float(np.median(drops)), np.round(drops, 2).tolist()))
    assert float(np.median(drops)) <= 2.0


# ---- behaviour: a rotating blob ----------------------------------------------------------------------------------------------
def _blob():
    """A jittered ball of fluid of radius 0.4 spinning at 6 rad/s about y, in zero gravity."""
    pts = scenes.jitter(scenes.block_lattice(16, 16, 16, S.R, origin=(-0.8, -0.8, -0.8)), S.R, 5)
    c = np.zeros(3)
    pts = pts[np.linalg.norm(pts - c, axis=1) <= 0.4].astype(F)
    vel = np.cross(np.array([0.0, 6.0, 0.0]), pts.astype(np.float64)).astype(F)
    return pts, vel


def _spin(eps, steps=100):
    pts, vel = _blob()
    w = LiquidWorld(particle_radius=S.R)
    fh = w.add_fluid(pts, velocities=vel)
    w.push_force(fh, *scenes.xsph_viscosity(0.5, 0.0))
    if eps:
        w.push_force(fh, *scenes.vorticity_confinement(eps))
    for _ in range(steps):
        w.step(S.DT, S.ZERO_G)
    p, v = w.read_fluid(fh)
    m = F(S.R) ** 3 * F(8.0 * 0.8) * F(1000.0)
    ke = 0.5 * float(m) * float((v.astype(np.float64) ** 2).sum())
    mean_w = None
    if eps:
        c = p.astype(np.float64).mean(0)
        rad = np.linalg.norm(p - c, axis=1)
        inner = rad <= 0.5 * np.quantile(rad, 0.5)
        mean_w = float(np.linalg.norm(w.debug(fh, "vorticity")[inner].astype(np.float64), axis=1).mean())
    return ke, mean_w, len(pts)


@pytest.mark.gpu
def test_vorticity_confinement_keeps_a_rotating_blob_spinning():
    res = {eps: _spin(eps) for eps in (0.0, 0.02, 0.1)}
    print("\nVORTICITY_BLOB " + json.dumps({"particles": res[0.0][2], "steps": 100, "dt": S.DT,
                                           "kinetic_energy": {str(e): r[0] for e, r in res.items()},
                                           "interior_mean_abs_omega": {str(e): r[1] for e, r in res.items() if e}}))
    ke = [res[e][0] for e in (0.0, 0.02, 0.1)]
    assert ke[0] < ke[1] < ke[2], ke


if __name__ == "__main__" and sys.argv[1:] == ["lifetime"]:
    _lifetime_child()
