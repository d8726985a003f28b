"""Fluid surface extraction on the GPU (include/sph.h sph_world_extract_surface, DESIGN.md section 15) against the float64
field and the float32 restatement of the polygonisation in oracle/ref64_surface.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref64_surface as S  # noqa: E402
from salva_b200 import DFSPHSolver, LiquidWorld, scenes  # noqa: E402
from salva_b200.liquid_world import Poly6Kernel, SphError, SpikyKernel  # noqa: E402

F = np.float32
R = 0.05
DT = 1.0 / 200.0
KINDS = {"cubic": (0, 0), "poly6": (1, 2)}


def _world(kind="cubic", deterministic=True):
    kd, kg = KINDS[kind]
    solver = DFSPHSolver(kernel_density=Poly6Kernel, kernel_gradient=SpikyKernel) if kd else None
    return LiquidWorld(solver=solver, particle_radius=R, deterministic=deterministic)


def _block(n=8, seed=3, origin=(0.0, 0.0, 0.0)):
    return scenes.jitter(scenes.block_lattice(n, n, n, R, origin=origin), R, seed)


def _tank_world(kind="cubic", n=8, volumes=None, second=False, deterministic=True):
    w = _world(kind, deterministic)
    f = w.add_fluid(_block(n), volumes=volumes)
    side = 2 * R * n + R
    g = w.add_fluid(_block(4, 9, origin=(0.1, 0.9, 0.1))) if second else None
    w.add_boundary(scenes.open_tank((-R, -R, -R), (side, 2 * side, side), R))
    return w, f, g


def _volumes(w, f, given):
    n = w.num_particles(f)
    return np.full(n, F(0.8 * (2 * R) ** 3)) if given is None else np.asarray(given, F)


def _check_field(w, fluids, vols, kind):
    phi, o, s = w.surface_field()
    dims = np.array(phi.shape[::-1])
    pos = np.concatenate([w.read_fluid(f)[0] for f in fluids])
    ref, bound = S.field64(pos, np.concatenate(vols), S.points(o, dims, s), float(w.h), KINDS[kind][0])
    err = np.abs(phi.reshape(-1).astype(np.float64) - ref)
    assert np.all(err <= bound), "phi off by %g > bound at %d points" % (float(err.max()), int((err > bound).sum()))
    assert phi.max() > 0.5
    return phi, o, dims, s


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("xysub", ["1", "2"])
@pytest.mark.parametrize("case", ["block", "two_fluids", "volumes", "clipped", "odd_spacing", "before_step"])
def test_field_within_the_float64_bound(case, kind, xysub, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", xysub)
    vols = None
    if case == "volumes":
        vols = (0.8 * (2 * R) ** 3 * np.random.default_rng(5).uniform(0.6, 1.4, 512)).astype(F)
    w, f, g = _tank_world(kind, volumes=vols, second=case == "two_fluids")
    if case != "before_step":
        for _ in range(3):
            w.step(DT)
    spacing = {"odd_spacing": 0.7 * R}.get(case, R)
    box = ((0.1, 0.05, 0.12), (0.5, 0.6, 0.45)) if case == "clipped" else None
    w.extract_surface(iso=0.6, spacing=spacing, fluids=[f], box=box, normals=True)
    phi, o, dims, s = _check_field(w, [f], [_volumes(w, f, vols)], kind)
    if box is not None:
        assert np.all(o <= np.asarray(box[0], F)) and np.all(o + (dims - 1) * s >= np.asarray(box[1], F) - s)
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_mesh_is_the_restatement_of_the_gpu_field(kind):
    w, f, _ = _tank_world(kind)
    for _ in range(5):
        w.step(DT)
    v, t, n = w.surface_mesh(iso=0.6, spacing=R)
    phi, o, s = w.surface_field()
    rv, rt = S.polygonise(phi, o, np.array(phi.shape[::-1]), s, 0.6)
    assert len(t) > 100
    assert np.array_equal(rt, t)
    assert np.array_equal(rv.view(np.uint32), v.view(np.uint32))
    # normals: within the float64 bound of -grad phi / |grad phi| where |grad phi| is well above its bound
    pos = w.read_fluid(f)[0]
    n64, m, gb = S.normals64(pos, _volumes(w, f, None), v, float(w.h), KINDS[kind][1])
    ok = m > 1000.0 * gb
    assert ok.mean() > 0.9
    dev = np.linalg.norm(n.astype(np.float64) - n64, axis=1)[ok]
    allowed = (2.0 * np.sqrt(3.0) * gb / m)[ok] + 1e-5
    assert np.all(dev <= allowed), float(dev.max())
    w.close()


def _closed_checks(v, t, label):
    assert len(t) > 0, label
    assert S.watertight_oriented(t), label
    comps = S.components(len(v), t)
    assert comps >= 1 and S.euler(len(v), t) == 2 * comps, (label, comps, S.euler(len(v), t))
    assert S.volume(v, t) > 0, label


@pytest.mark.gpu
def test_basic3_after_50_steps_is_watertight_oriented_and_encloses_the_float64_volume():
    sc = scenes.scene_c1()
    w = LiquidWorld(particle_radius=sc["particle_radius"])
    (f,), _ = scenes.populate(w, sc)
    for _ in range(50):
        w.step(sc["dt"])
    v, t, _ = w.surface_mesh(iso=0.6, spacing=R, normals=False)
    _closed_checks(v, t, "basic3")
    phi, o, s = w.surface_field()
    dims = np.array(phi.shape[::-1])
    ref, bound = S.field64(w.read_fluid(f)[0], F(0.8 * (2 * R) ** 3), S.points(o, dims, s), float(w.h))
    assert np.all(np.abs(phi.reshape(-1) - ref) <= bound)
    v64, t64 = S.polygonise(ref, o, dims, s, 0.6, dtype=np.float64)
    tol = S.volume_bound(phi, ref, bound, dims, float(s), 0.6, S.area(v, t))
    assert abs(S.volume(v, t) - S.volume(v64, t64)) <= tol, (S.volume(v, t), S.volume(v64, t64), tol)
    w.close()


@pytest.mark.gpu
def test_c2_full_size_is_watertight_and_oriented():
    sc = scenes.scene_c2()
    w = LiquidWorld(particle_radius=sc["particle_radius"])
    scenes.populate(w, sc)
    for _ in range(5):
        w.step(sc["dt"])
    v, t, _ = w.surface_mesh(iso=0.6, normals=False)
    _closed_checks(v, t, "C2")
    w.close()


def _twin(with_edits):
    w, f, _ = _tank_world(n=10)
    if with_edits:
        w.add_sink(f, (-10.0, -10.0, -10.0), (10.0, 0.06, 10.0))
        w.add_source(f, _block(3, 4, origin=(0.3, 1.2, 0.3)), interval=4)
    return w, f


@pytest.mark.gpu
@pytest.mark.parametrize("with_edits", [False, True])
def test_extraction_does_not_change_the_steps(with_edits):
    a, fa = _twin(with_edits)
    b, fb = _twin(with_edits)
    for k in range(20):
        a.step(DT)
        b.step(DT)
        a.extract_surface(iso=0.6, spacing=R if k % 2 else 0.7 * R, normals=bool(k % 3))
        assert a.snapshot() == b.snapshot()
        assert [np.array_equal(x, y) for x, y in zip(a.read_fluid(fa), b.read_fluid(fb))] == [True, True]
        assert np.array_equal(a.read_ids(fa), b.read_ids(fb))
        assert a.step_records() == b.step_records()
    if not with_edits:
        for w in (a, b):
            w.step_many(DT, 8)
        a.extract_surface()
        for w in (a, b):
            w.step_many(DT, 8)
        assert a.step_records() == b.step_records()
        assert any(r["on_device"] for r in a.step_records())
        assert a.stats()["kernel_launches"] == b.stats()["kernel_launches"]
        assert a.snapshot() == b.snapshot()
    a.close()
    b.close()


@pytest.mark.gpu
def test_extraction_is_deterministic_and_independent_of_slot_order():
    pts = _block(9, 11)
    ids = np.arange(len(pts), dtype=np.uint32)
    perm = np.random.default_rng(2).permutation(len(pts))
    out = []
    for order in (np.arange(len(pts)), perm):
        w = _world()
        f = w.add_fluid(pts[order])
        w.set_ids(f, ids[order])
        for _ in range(2):
            v, t, n = w.surface_mesh(iso=0.55, spacing=0.8 * R)
            out.append((v.tobytes(), t.tobytes(), n.tobytes(), w.surface_field()[0].tobytes()))
        w.close()
    assert out[0] == out[1] == out[2] == out[3]


@pytest.mark.gpu
def test_refusals_change_nothing_and_keep_the_previous_mesh():
    w, f, g = _tank_world(second=True)
    w.step(DT)
    v0, t0, n0 = w.surface_mesh(iso=0.6)
    phi0 = w.surface_field()[0]

    def refused(**kw):
        with pytest.raises(SphError) as e:
            w.extract_surface(**kw)
        assert e.value.status == 1
        v, t, n = w.read_surface()
        assert np.array_equal(v, v0) and np.array_equal(t, t0) and np.array_equal(n, n0)
        assert np.array_equal(w.surface_field()[0], phi0)

    refused(iso=float("nan"))
    refused(iso=0.0)
    refused(spacing=-1.0)
    refused(spacing=float("inf"))
    refused(box=((0.0, 1.0, 0.0), (1.0, 0.0, 1.0)))           # lo > hi on one axis only
    refused(box=((0.0, float("nan"), 0.0), (1.0, 1.0, 1.0)))
    refused(fluids=[f, f])
    refused(fluids=[f + (7 << 16)])
    mask = np.zeros(w.num_particles(f), np.uint8)
    mask[0] = 1
    w.delete_particles(f, mask)                                 # a pending host edit
    refused()
    w.step(DT)
    nv, nt = w.extract_surface(iso=0.6)
    # caps and normals
    L = w._L
    import ctypes as C
    vv = np.empty((nv, 3), F)
    tt = np.empty((nt, 3), np.uint32)
    assert L.sph_world_read_surface(w._w, vv.ctypes.data_as(C.POINTER(C.c_float)), None, nv - 1, tt.ctypes.data_as(C.POINTER(C.c_uint32)), nt) == 1
    assert L.sph_world_read_surface(w._w, vv.ctypes.data_as(C.POINTER(C.c_float)), None, nv, tt.ctypes.data_as(C.POINTER(C.c_uint32)), nt - 1) == 1
    w.extract_surface(iso=0.6, normals=False)
    with pytest.raises(SphError):
        w.read_surface(normals=True)
    # mapped views equal the read copies
    import torch
    v, t, _ = w.read_surface()
    mv, mt, mn = w.map_surface()
    assert mn is None
    assert np.array_equal(torch.as_tensor(mv, device="cuda").cpu().numpy(), v)
    assert np.array_equal(torch.as_tensor(mt, device="cuda").cpu().numpy().astype(np.uint32), t)
    # a host-force callback cannot extract
    seen = []

    def cb(*_):
        try:
            w.extract_surface()
            seen.append("ran")
        except SphError:
            seen.append("refused")
    w.push_host_force(g, cb)
    w.step(DT)
    assert seen == ["refused"]
    w.close()


@pytest.mark.gpu
def test_empty_selection_and_before_the_first_step():
    w = _world()
    assert w.extract_surface() == (0, 0)
    phi, o, s = w.surface_field()
    assert phi.size == 0
    f = w.add_fluid(np.zeros((0, 3), F))
    assert w.extract_surface(fluids=[f]) == (0, 0)
    g = w.add_fluid(_block(6))
    nv, nt = w.extract_surface(fluids=[g])  # before the first step: the positions given
    assert nv > 0 and nt > 0
    v, t, _ = w.read_surface()
    _closed_checks(v, t, "before the first step")
    assert w.extract_surface(fluids=[f]) == (0, 0)
    w.close()


def _lifetime_child():
    import torch
    free = []
    for _ in range(9):
        w, f, _ = _tank_world(n=40)
        w.step(DT)
        w.extract_surface(spacing=0.5 * R)
        w.close()
        free.append(torch.cuda.mem_get_info()[0])
    print("LIFETIME " + json.dumps(free))


@pytest.mark.gpu
def test_destroyed_world_returns_the_surface_memory():
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "lifetime"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    free = json.loads([x for x in r.stdout.splitlines() if x.startswith("LIFETIME ")][-1][len("LIFETIME "):])
    drops = -np.diff(np.asarray(free, np.float64)) / float(1 << 20)
    assert float(np.median(drops)) <= 2.0, drops.tolist()


if __name__ == "__main__" and sys.argv[1:] == ["lifetime"]:
    _lifetime_child()
