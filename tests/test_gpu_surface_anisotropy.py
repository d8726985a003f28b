"""Anisotropic fluid surfaces on the GPU (include/sph.h sph_world_extract_surface_anisotropic, DESIGN.md section 17) against
the float64 restatement in oracle/ref64_anisotropy.py: each pass on its own inputs (ellipsoids from the positions, the field
from the device's own ellipsoid rows, the mesh from the device's own field)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref64_anisotropy as A  # noqa: E402
from oracle import ref64_surface as S  # noqa: E402
from salva_b200 import DFSPHSolver, LiquidWorld, SurfaceAnisotropy, scenes  # noqa: E402
from salva_b200.liquid_world import Poly6Kernel, SphError, SpikyKernel  # noqa: E402

F = np.float32
R = 0.05
DT = 1.0 / 200.0
KINDS = {"cubic": (0, 0), "poly6": (1, 2)}
V0 = F(0.8 * (2 * R) ** 3)
AN = SurfaceAnisotropy(max_ratio=4.0, isolated_radius=0.5)  # stretched kernels: every branch of the ellipsoid pass
DEF = SurfaceAnisotropy()  # the defaults: what the mesh-quality checks hold


def _world(kind="cubic"):
    kd, _ = KINDS[kind]
    solver = DFSPHSolver(kernel_density=Poly6Kernel, kernel_gradient=SpikyKernel) if kd else None
    return LiquidWorld(solver=solver, particle_radius=R, deterministic=True)


def _block(n=8, seed=3, origin=(0.0, 0.0, 0.0)):
    return scenes.jitter(scenes.block_lattice(n, n, n, R, origin=origin), R, seed)


def _tank(w, n=8):
    side = 2 * R * n + R
    w.add_boundary(scenes.open_tank((-R, -R, -R), (side, 2 * side, side), R))


def _line_and_lone():
    """A straight line, a lone particle, and particles with exactly N_eps - 1 and N_eps neighbours at |x_ij|^2 = h^2."""
    h = F(4 * R)
    line = np.zeros((20, 3), F)
    line[:, 0] = np.arange(20, dtype=F) * F(R)
    line += F(2.0)
    lone = np.array([[3.0, 3.0, 3.0]], F)
    out = [line, lone]
    for k, o in ((5, 4.0), (6, 5.0)):
        dirs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], F)
        nb = [np.array([F(0.5) * h, 0, 0], F)] + list(dirs[: k - 1] * h)
        out.append((np.concatenate([np.zeros((1, 3), F), np.asarray(nb, F)]) + F(o)).astype(F))
    return np.concatenate(out)


def _check_ellipsoids(w, fluids):
    """The selected fluids' rows against the float64 ellipsoids of all their particles together."""
    pos = np.concatenate([w.read_fluid(f)[0] for f in fluids])
    rows = [w.surface_ellipsoids(f) for f in fluids]
    c, ax = np.concatenate([r[0] for r in rows]), np.concatenate([r[1] for r in rows])
    assert len(c) == len(pos) and all(len(r[0]) == w.num_particles(f) for r, f in zip(rows, fluids))
    el = A.ellipsoids64(pos, float(w.h), AN.smoothing, AN.max_ratio, AN.isolated_radius, AN.min_neighbours)
    fin = el["finite"]
    ce = np.abs(c[fin].astype(np.float64) - el["centre"][fin])
    assert np.all(ce <= el["centre_bound"][fin][:, None]), float(ce.max())
    e, a = ax[:, :, :3].astype(np.float64), ax[:, :, 3].astype(np.float64)
    M = np.einsum("nki,nk,nkj->nij", e, a * a, e)
    me = np.sqrt(((M - el["M"]) ** 2).sum(axis=(1, 2)))
    ok = fin & np.isfinite(el["M_bound"])
    assert np.all(me[ok] <= el["M_bound"][ok]), float((me[ok] / el["M_bound"][ok]).max())
    h = float(w.h)
    af = a[fin]
    assert np.all(af[:, 0] >= af[:, 1]) and np.all(af[:, 1] >= af[:, 2])
    iso_r = float(F(AN.isolated_radius) * F(h))
    aniso_ok = (af[:, 0] == F(h)) & (af >= h / AN.max_ratio * (1 - 1e-6)).all(axis=1)
    assert np.all(aniso_ok | (af == F(iso_r)).all(axis=1))
    assert np.array_equal(af[:, 0] == F(h), el["aniso"][fin])
    G = np.einsum("nki,nkj->nij", e[fin], e[fin])
    assert np.abs(G - np.eye(3)).max() <= 1e-5
    assert np.array_equal(c[~fin].view(np.uint32), pos[~fin].view(np.uint32)) and np.all(ax[~fin] == 0)
    return pos, c, ax


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("xysub", ["1", "2"])
@pytest.mark.parametrize("case", ["block", "two_fluids", "line_and_lone", "before_step", "non_finite"])
def test_ellipsoids_field_mesh_and_normals_within_the_float64_bounds(case, kind, xysub, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", xysub)
    w = _world(kind)
    vols = None
    if case == "two_fluids":
        vols = (V0 * np.random.default_rng(5).uniform(0.6, 1.4, 512)).astype(F)
    pts = _line_and_lone() if case == "line_and_lone" else _block()
    f = w.add_fluid(pts, volumes=vols)
    g = w.add_fluid(_block(4, 9, origin=(0.1, 0.9, 0.1))) if case == "two_fluids" else None
    if case != "line_and_lone":
        _tank(w)
    if case == "non_finite":
        p, v = w.read_fluid(f)
        p[7] = np.nan
        p[9, 1] = np.inf
        w.write_fluid(f, p, v)
    if case not in ("before_step", "line_and_lone", "non_finite"):
        for _ in range(3):
            w.step(DT)
    fluids = [f, g] if g is not None else [f]
    nv, nt = w.extract_surface(iso=0.6, spacing=R, fluids=fluids, normals=True, anisotropy=AN)
    assert nt > 0
    pos, c, ax = _check_ellipsoids(w, fluids)
    vol = np.concatenate([np.full(w.num_particles(fl), V0) if vv is None else vv for fl, vv in zip(fluids, [vols, None])])
    # the field from the device's own ellipsoid rows
    phi, o, s = w.surface_field()
    dims = np.array(phi.shape[::-1])
    h = float(w.h)
    ref, bound = A.field64(c, ax, vol, S.points(o, dims, s), h, KINDS[kind][0])
    err = np.abs(phi.reshape(-1).astype(np.float64) - ref)
    assert np.all(err <= bound), "phi off by %g > bound at %d points" % (float(err.max()), int((err > bound).sum()))
    # the mesh from the device's own field, bit for bit; normals within their bound
    v, t, n = w.read_surface()
    rv, rt = S.polygonise(phi, o, dims, s, 0.6)
    assert np.array_equal(rt, t) and np.array_equal(rv.view(np.uint32), v.view(np.uint32))
    n64, m, gb = A.normals64(c, ax, vol, v, h, KINDS[kind][1])
    ok = m > 1000.0 * gb
    assert ok.mean() > 0.5  # a thin line's vertices have ill-conditioned gradients; every well-conditioned one is checked
    dev = np.linalg.norm(n.astype(np.float64) - n64, axis=1)[ok]
    assert np.all(dev <= (2.0 * np.sqrt(3.0) * gb / m)[ok] + 1e-5), float(dev.max())
    w.close()


def _closed_checks(v, t, label, components=None, genus0=True):
    """Watertight, oriented, enclosing a positive volume; with `components`, no more pieces than the isotropic mesh (no
    inner shells); with genus0, V - E + F = 2 per piece."""
    assert len(t) > 0, label
    assert S.watertight_oriented(t), label
    comps = S.components(len(v), t)
    assert comps >= 1, label
    if genus0:
        assert S.euler(len(v), t) == 2 * comps, (label, comps, S.euler(len(v), t))
    if components is not None:
        assert comps <= components, (label, comps, components)
    assert S.volume(v, t) > 0, label


@pytest.mark.gpu
def test_basic3_after_50_steps_is_watertight_oriented_and_encloses_the_float64_volume():
    sc = scenes.scene_c1()
    w = LiquidWorld(particle_radius=sc["particle_radius"])
    (f,), _ = scenes.populate(w, sc)
    for _ in range(50):
        w.step(sc["dt"])
    vi, ti, _ = w.surface_mesh(iso=0.6, spacing=R, normals=False)
    v, t, _ = w.surface_mesh(iso=0.6, spacing=R, normals=False, anisotropy=DEF)
    # Mid-splash the default mesh has 7 pieces, one of genus 1, where the isotropic mesh has 3 (DESIGN.md section 17):
    # neither genus nor the piece count is compared here, only what the mesh must be in every case.
    _closed_checks(v, t, "basic3", genus0=False)
    c, ax = w.surface_ellipsoids(f)
    phi, o, s = w.surface_field()
    dims = np.array(phi.shape[::-1])
    ref, bound = A.field64(c, ax, V0, S.points(o, dims, s), float(w.h))
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
    vi, ti, _ = w.surface_mesh(iso=0.6, normals=False)
    v, t, _ = w.surface_mesh(iso=0.6, normals=False, anisotropy=DEF)
    _closed_checks(v, t, "C2", components=S.components(len(vi), ti))
    w.close()


def _twin():
    w = _world()
    f = w.add_fluid(_block(10))
    _tank(w, 10)
    return w, f


@pytest.mark.gpu
def test_extraction_changes_neither_the_steps_nor_the_isotropic_extraction():
    a, fa = _twin()
    b, fb = _twin()
    for k in range(12):
        a.step(DT)
        b.step(DT)
        a.extract_surface(iso=0.6, spacing=R, normals=bool(k % 2), anisotropy=AN)
        # an isotropic extraction after an anisotropic one equals one made without it
        ma, mb = a.surface_mesh(iso=0.6, spacing=R), b.surface_mesh(iso=0.6, spacing=R)
        assert all(np.array_equal(x, y) for x, y in zip(ma, mb))
        assert np.array_equal(a.surface_field()[0], b.surface_field()[0])
        assert len(a.surface_ellipsoids(fa)[0]) == 0
        assert a.snapshot() == b.snapshot()
        assert [np.array_equal(x, y) for x, y in zip(a.read_fluid(fa), b.read_fluid(fb))] == [True, True]
        assert a.step_records() == b.step_records()
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
        inv = np.argsort(order)
        for _ in range(2):
            v, t, n = w.surface_mesh(iso=0.55, spacing=0.8 * R, anisotropy=AN)
            c, ax = w.surface_ellipsoids(f)
            out.append((v.tobytes(), t.tobytes(), n.tobytes(), w.surface_field()[0].tobytes(), c[inv].tobytes(), ax[inv].tobytes()))
        w.close()
    assert out[0] == out[1] == out[2] == out[3]


@pytest.mark.gpu
def test_refusals_change_nothing_and_keep_the_previous_mesh_and_ellipsoids():
    w = _world()
    f = w.add_fluid(_block())
    g = w.add_fluid(_block(4, 9, origin=(0.1, 0.9, 0.1)))
    _tank(w)
    w.step(DT)
    v0, t0, n0 = w.surface_mesh(iso=0.6, anisotropy=AN)
    phi0 = w.surface_field()[0]
    c0, a0 = w.surface_ellipsoids(f)
    assert len(c0) == w.num_particles(f) and len(w.surface_ellipsoids(g)[0]) == w.num_particles(g)

    def refused(**kw):
        an = kw.pop("an", AN)
        with pytest.raises(SphError) as e:
            w.extract_surface(anisotropy=an, **kw)
        assert e.value.status == 1
        v, t, n = w.read_surface()
        assert np.array_equal(v, v0) and np.array_equal(t, t0) and np.array_equal(n, n0)
        assert np.array_equal(w.surface_field()[0], phi0)
        c, a = w.surface_ellipsoids(f)
        assert np.array_equal(c, c0) and np.array_equal(a, a0)

    refused(iso=float("nan"))
    refused(spacing=-1.0)
    refused(box=((0.0, 1.0, 0.0), (1.0, 0.0, 1.0)))
    refused(fluids=[f, f])
    for bad in (dict(smoothing=float("nan")), dict(smoothing=1.5), dict(smoothing=-0.1), dict(max_ratio=0.5),
                dict(max_ratio=float("inf")), dict(max_ratio=float("nan")), dict(max_ratio=1000.5), dict(isolated_radius=0.0),
                dict(isolated_radius=9e-4), dict(isolated_radius=1.5), dict(isolated_radius=float("nan"))):
        refused(an=SurfaceAnisotropy(**bad))
    mask = np.zeros(w.num_particles(f), np.uint8)
    mask[0] = 1
    w.delete_particles(f, mask)
    refused()
    w.step(DT)
    # only the selected fluid has rows; the mapped rows equal the read ones
    w.extract_surface(iso=0.6, fluids=[g], anisotropy=AN)
    assert len(w.surface_ellipsoids(f)[0]) == 0
    import torch
    c, a = w.surface_ellipsoids(g)
    mc, ma = w.map_surface_ellipsoids(g)
    assert np.array_equal(torch.as_tensor(mc, device="cuda").cpu().numpy(), c)
    assert np.array_equal(torch.as_tensor(ma, device="cuda").cpu().numpy(), a)
    w.close()


@pytest.mark.gpu
def test_empty_selection_and_before_the_first_step():
    w = _world()
    assert w.extract_surface(anisotropy=AN) == (0, 0)
    f = w.add_fluid(np.zeros((0, 3), F))
    assert w.extract_surface(fluids=[f], anisotropy=AN) == (0, 0)
    assert len(w.surface_ellipsoids(f)[0]) == 0
    g = w.add_fluid(_block(6))
    nv, nt = w.extract_surface(fluids=[g], anisotropy=AN)
    assert nv > 0 and nt > 0
    v, t, _ = w.read_surface()
    _closed_checks(v, t, "before the first step")
    _check_ellipsoids(w, [g])
    w.close()


@pytest.mark.gpu
def test_the_largest_allowed_ratio_keeps_a_planar_neighbourhood_finite():
    """k_r = 1000 on a plane of particles (s3 = 0): a3 = h / 1000, and phi stays finite."""
    w = _world()
    g = np.stack(np.meshgrid(np.arange(12), np.arange(12), indexing="ij"), -1).reshape(-1, 2).astype(F) * F(2 * R)
    f = w.add_fluid(np.stack([g[:, 0], np.full(len(g), F(0.5)), g[:, 1]], 1).astype(F))
    w.extract_surface(iso=0.6, spacing=R, anisotropy=SurfaceAnisotropy(max_ratio=1000.0, isolated_radius=0.001))
    phi = w.surface_field()[0]
    _, ax = w.surface_ellipsoids(f)
    assert np.all(np.isfinite(phi)) and phi.max() > 0
    assert np.all(ax[:, :, 3] > 0) and ax[:, 2, 3].min() >= F(w.h) / F(1000.0) * F(1 - 1e-6)
    w.close()


def _settled_pool():
    w = _world()
    f = w.add_fluid(scenes.jitter(scenes.block_lattice(20, 5, 20, R), R, 5))
    side = 2 * R * 20 + R
    w.add_boundary(scenes.open_tank((-R, -R, -R), (side, 1.0, side), R))
    for _ in range(150):
        w.step(DT)
    return w, f


@pytest.mark.gpu
def test_a_settled_pool_is_flatter_with_the_default_anisotropy():
    """The top-face vertices (normal within 10 degrees of +y, more than 2 h from the walls) of the device meshes."""
    w, f = _settled_pool()
    pos = w.read_fluid(f)[0]
    h = float(w.h)
    pmin, pmax = pos.min(axis=0), pos.max(axis=0)
    out = []
    for an in (None, DEF):
        v, t, n = w.surface_mesh(iso=0.6, spacing=R, anisotropy=an)
        sel = (n[:, 1] > np.cos(np.radians(10.0))) & (v[:, 0] > pmin[0] + 2 * h) & (v[:, 0] < pmax[0] - 2 * h) \
            & (v[:, 2] > pmin[2] + 2 * h) & (v[:, 2] < pmax[2] - 2 * h) & (v[:, 1] > pmax[1] - h)
        assert sel.sum() > 100
        out.append((float(np.std(v[sel, 1].astype(np.float64))), S.components(len(v), t)))
    print("settled pool top-face height std: isotropic %.3e, default anisotropy %.3e, ratio %.3f" % (out[0][0], out[1][0], out[1][0] / out[0][0]))
    assert out[1][0] < out[0][0]
    assert out[1][1] == out[0][1]
    w.close()


def _lifetime_child():
    import torch
    free = []
    for _ in range(9):
        w = _world()
        w.add_fluid(_block(24))
        w.step(DT)
        w.extract_surface(spacing=0.5 * R, anisotropy=AN)
        w.close()
        free.append(torch.cuda.mem_get_info()[0])
    print("LIFETIME " + json.dumps(free))


@pytest.mark.gpu
def test_destroyed_world_returns_the_anisotropic_surface_memory():
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "lifetime"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    free = json.loads([x for x in r.stdout.splitlines() if x.startswith("LIFETIME ")][-1][len("LIFETIME "):])
    drops = -np.diff(np.asarray(free, np.float64)) / float(1 << 20)
    assert float(np.median(drops)) <= 2.0, drops.tolist()


if __name__ == "__main__" and sys.argv[1:] == ["lifetime"]:
    _lifetime_child()
