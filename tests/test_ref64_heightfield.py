"""CPU checks of heightfield colliders: the float32 restatement (salva_b200/contact_sampling.py, which the device matches bit
for bit) against the float64 reference oracle/ref64_heightfield.py, closed forms, plausible bugs the bounds must catch, and
the C++ example's build."""
import os
import subprocess

import numpy as np
import pytest

from oracle import ref64_colliders as rc
from oracle import ref64_heightfield as rh
from salva_b200 import contact_sampling as cs

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def heightfield3_heights(n=41):
    """heightfield3.rs:46-61: 3.0 on the rim, sin(i * 12 / 40) + cos(j * 12 / 40) inside (float32, as the examples compute)."""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    x, z = (i * F(12.0) / F(n - 1)).astype(F), (j * F(12.0) / F(n - 1)).astype(F)
    h = (np.sin(x) + np.cos(z)).astype(F)
    h[[0, -1], :] = 3.0
    h[:, [0, -1]] = 3.0
    return h


def _points(rng, g, n):
    """Points inside, above, below and beyond the rim, on cell edges, on diagonals and on vertices of grid g."""
    hx, hz = float(g["hx"]), float(g["hz"])
    ylo, yhi = float(g["ylo"]), float(g["yhi"])
    nr, nc = g["nrows"], g["ncols"]
    rand = np.stack([rng.uniform(-1.3 * hx, 1.3 * hx, n), rng.uniform(ylo - 1.0, yhi + 1.0, n), rng.uniform(-1.3 * hz, 1.3 * hz, n)], 1)
    j, i = rng.integers(0, nc, n), rng.integers(0, nr, n)
    xs = rh.grid32(j, nc - 1, g["hx"], g["dx"])
    zs = rh.grid32(i, nr - 1, g["hz"], g["dz"])
    t = rng.uniform(0, 1, n)
    y = rng.uniform(ylo - 0.5, yhi + 0.5, n)
    vertex = np.stack([xs, y, zs], 1)
    edge = np.stack([xs, y, rng.uniform(-hz, hz, n)], 1)
    jd, id_ = np.minimum(j, nc - 2), np.minimum(i, nr - 2)
    x0, z1 = rh.grid32(jd, nc - 1, g["hx"], g["dx"]), rh.grid32(id_ + 1, nr - 1, g["hz"], g["dz"])
    x1, z0 = rh.grid32(jd + 1, nc - 1, g["hx"], g["dx"]), rh.grid32(id_, nr - 1, g["hz"], g["dz"])
    diag = np.stack([x0 + t * (x1 - x0), y, z1 + t * (z0 - z1)], 1)
    return np.concatenate([rand, vertex, edge, diag]).astype(F)


def _random_fields():
    rng = np.random.default_rng(5)
    yield rng.normal(0, 0.6, (9, 13)).astype(F), (3.0, 1.3, 2.0)
    yield rng.normal(0, 3.0, (6, 5)).astype(F), (1.0, 0.5, 1.5)  # rugged: slopes far steeper than the cells
    yield rng.uniform(2.0, 3.0, (2, 2)).astype(F), (0.7, 1.0, 0.4)
    yield heightfield3_heights(), (12.0, 1.0, 12.0)


@pytest.mark.parametrize("case", range(4))
def test_ring_search_equals_the_all_triangle_loop(case):
    """Within the cap, the ring search's closest point is the float64 loop's over every triangle, within its bound, outside
    the counted exclusions; points are inside, above, below and beyond the rim and on edges, diagonals and vertices."""
    H, scale = list(_random_fields())[case]
    g = cs.hf_grid(H, scale)
    fld = rh.field(H, scale)
    l = _points(np.random.default_rng(case), g, 500)
    cap = F(0.9)
    q, d2, found = cs.hf_project_local(g, l, cap)
    q64, eq, D, eD, _, amb_c, amb_r = rh.project64(fld, l.astype(np.float64), 0.0)
    within = D + eD < float(cap)
    assert found[within].all()
    ok = within & ~amb_c & ~amb_r
    r = np.abs(q[ok] - q64[ok]).max(axis=1) / eq[ok]
    assert r.max(initial=0) <= 1.0, r.max()
    assert np.abs(np.sqrt(d2[ok].astype(np.float64)) - D[ok]).max(initial=0) <= (eD[ok] + 1e-6 * D[ok]).max(initial=0)
    assert (amb_c | amb_r)[:500][within[:500]].mean() < 0.01  # the random points; the others sit on region boundaries
    assert within.sum() > 300


def test_flat_field_projects_down_inside_and_onto_the_rim_outside():
    H = np.full((5, 7), 0.25, F)
    g = cs.hf_grid(H, (3.0, 2.0, 2.0))  # y = 0.5
    l = np.array([[0.3, 1.0, -0.2], [-1.25, -0.75, 0.5], [0.0, 0.5, 0.0], [2.0, 0.75, 0.25], [-1.75, 0.0, 1.5]], F)
    q, d2, found = cs.hf_project_local(g, l, F(2.0))
    want = np.array([[0.3, 0.5, -0.2], [-1.25, 0.5, 0.5], [0.0, 0.5, 0.0], [1.5, 0.5, 0.25], [-1.5, 0.5, 1.0]], F)
    assert found.all()
    np.testing.assert_allclose(q, want, atol=2e-7)
    np.testing.assert_allclose(d2, ((l - want) ** 2).sum(1), rtol=1e-6)


def test_tilted_plane_gives_the_plane_projection():
    nr, nc, sx, sz = 6, 8, 2.0, 1.5
    x = rh.grid32(np.arange(nc), nc - 1, F(sx) * F(0.5), F(sx) / F(nc - 1))
    z = rh.grid32(np.arange(nr), nr - 1, F(sz) * F(0.5), F(sz) / F(nr - 1))
    H = (0.3 * x[None, :] - 0.2 * z[:, None]).astype(F)  # y = 0.3 x - 0.2 z
    g = cs.hf_grid(H, (sx, 1.0, sz))
    rng = np.random.default_rng(2)
    l = np.stack([rng.uniform(-0.5, 0.5, 200), rng.uniform(-0.4, 0.4, 200), rng.uniform(-0.4, 0.4, 200)], 1).astype(F)
    n = np.array([0.3, -1.0, -0.2]) / np.linalg.norm([0.3, -1.0, -0.2])
    s = (l.astype(np.float64) @ n)  # signed distance to the plane 0.3 x - y - 0.2 z = 0
    want = l - s[:, None] * n
    inside = (np.abs(want[:, 0]) < 0.9 * sx / 2) & (np.abs(want[:, 2]) < 0.9 * sz / 2)
    q, d2, _ = cs.hf_project_local(g, l, F(1.0))
    assert inside.sum() > 150
    # coplanar neighbours' squared distances differ by |s| delta^2 / 2 for an in-plane offset delta, below float32's
    # resolution of |s|^2 until delta reaches about |s| sqrt(u): either triangle may win within that
    tol = 4 * 2.0 ** -12 * np.abs(s) + 2e-6
    assert np.all(np.abs(q[inside] - want[inside]).max(axis=1) <= tol[inside])
    assert np.median(np.abs(q[inside] - want[inside])) < 2e-7


def _scenes():
    """(pos, vel, colliders, h, radius, dt) of a rotated, translated field on a dynamic body with angular velocity, with fluid
    above, below and beyond the rim, overlapping a ball collider of the next slot; and heightfield3's ground under a block."""
    rng = np.random.default_rng(9)
    H = (rng.normal(0, 0.3, (9, 13)) + 0.5).astype(F)
    hf = dict(kind=rh.HEIGHTFIELD, params=(), heights=H, scale=(3.0, 1.3, 2.0),
              **rc._state((0.1, 0.2, -0.1), rc.rot(0.3, 0.2, 0.1), rc.BODY_DYNAMIC, (0.1, 0, 0), (0, 1, 0.5), (0.0, 0.3, 0.0)))
    ball = dict(kind=rc.BALL, params=(0.3,), **rc._state((0.5, 0.6, 0.2), None, rc.BODY_DYNAMIC, (0, -1, 0), (1, 0, 0)))
    pos = (rng.uniform(-1, 1, (3000, 3)) * np.array([2.0, 1.0, 1.5]) + np.array([0, 0.8, 0])).astype(F)
    vel = rng.normal(0, 1, pos.shape).astype(F)
    yield pos, vel, [hf, ball], 0.2, 0.05, 0.004
    yield pos, vel, [ball, hf], 0.2, 0.05, 0.008
    g = dict(kind=rh.HEIGHTFIELD, params=(), heights=heightfield3_heights(), scale=(12.0, 1.0, 12.0), **rc._state((0, 0, 0), None, rc.BODY_FIXED))
    block = rc.lattice((20, 6, 20), 0.3, (-3.0, 1.4, -3.0), seed=4, amplitude=0.2)
    vb = np.tile(np.array([0, -3.0, 0], F), (len(block), 1))
    yield block, vb, [g], 0.6, 0.15, 0.005


@pytest.mark.parametrize("case", range(3))
def test_restatement_within_the_float64_bounds(case):
    pos, vel, cols, h, r, dt = list(_scenes())[case]
    p32, v32, samples = cs.contact_sample(pos, vel, cols, dt, h, r)
    res = rh.contact64(pos, vel, cols, dt, h, r)
    w = rc.check_restatement(res, p32, v32, samples)
    assert max(w.values()) <= 1.0, w
    k = [c["kind"] for c in cols].index(rh.HEIGHTFIELD)
    assert len(samples[k][0]) > 200
    excluded = sum(v for key, v in res.reasons.items() if key in ("triangle_choice", "region", "depth_cut"))
    assert excluded <= 0.01 * res.hf_candidates, (res.reasons, res.hf_candidates)
    if cols[0]["kind"] == rh.HEIGHTFIELD:  # nothing pushes before the ball: the heightfield itself never pushes
        assert np.array_equal(p32, cs.contact_sample(pos, vel, cols[1:], dt, h, r)[0])


@pytest.mark.parametrize("mutant", rh.MUTANTS)
def test_reference_mutants_fail_the_bounds(mutant):
    pos, vel, cols, h, r, dt = list(_scenes())[0]
    if mutant == "uncentred_aabb":  # a field far from y = 0: its AABB's centre term moves the whole box
        cols = [dict(cols[0], heights=cols[0]["heights"] + F(4.0), translation=np.array([0.1, -5.0, -0.1], F))]
    p32, v32, samples = cs.contact_sample(pos, vel, cols, dt, h, r)
    res = rh.contact64(pos, vel, cols, dt, h, r, mutant=mutant)
    w = rc.check_restatement(res, p32, v32, samples)
    assert max(w.values()) > 1.0, (mutant, w)


def _tie_field():
    """Two spikes at (row 1, col 0) and (row 1, col 2) of a dyadic field; the point above vertex (1, 1) at the spikes' height
    is equidistant, exactly, from their slopes toward it: the left one comes first in parry's order, the point's own cell
    holds the right one."""
    H = np.zeros((3, 4), F)
    H[1, 0] = H[1, 2] = 1.0
    return H, (3.0, 1.0, 2.0)  # dx = dz = 1


def test_search_bugs_fail_the_bounds(monkeypatch):
    """The float32 search with no margin (ring r taken at r dmin) or ties taken in visit order fails the float64 bounds."""
    H, scale = _tie_field()
    g = cs.hf_grid(H, scale)
    l = np.array([[-0.5, 1.0, 0.0]], F)  # above vertex (1, 1)
    q64, eq, _, _, _, amb_c, _ = rh.project64(rh.field(H, scale), l.astype(np.float64), 0.0)
    q, _, _ = cs.hf_project_local(g, l, F(0.9))
    assert not amb_c[0] and np.abs(q - q64).max() <= eq[0]
    assert q64[0, 0] < l[0, 0]  # parry's order: the left slope
    monkeypatch.setattr(cs, "_beats", lambda d, t, best, bidx: d < best)
    qm, _, _ = cs.hf_project_local(g, l, F(0.9))
    assert np.abs(qm - q64).max() > eq[0]
    monkeypatch.undo()

    H, scale = list(_random_fields())[1]
    g = cs.hf_grid(H, scale)
    fld = rh.field(H, scale)
    l = _points(np.random.default_rng(11), g, 2000)
    q64, eq, D, eD, _, amb_c, amb_r = rh.project64(fld, l.astype(np.float64), 0.0)
    ok = (D + eD < 0.9) & ~amb_c & ~amb_r
    monkeypatch.setattr(cs, "_ring_gap", lambda r, g, margin: F(r) * g["dmin"])
    qm, _, _ = cs.hf_project_local(g, l, F(0.9))
    assert (np.abs(qm - q64).max(axis=1)[ok] > eq[ok]).any()


def test_heightfield_contact_example_builds_and_fails_loudly_without_cuda(tmp_path):
    import torch
    exe = str(tmp_path / "heightfield_contact3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "heightfield_contact3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    r = subprocess.run([exe, "1"], capture_output=True, text=True)
    assert r.returncode == 2 and "no CPU fallback" in r.stderr
