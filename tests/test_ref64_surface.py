"""The float32 restatement of the surface extractor's polygonisation (oracle/ref64_surface.py) on analytic fields, and the
mutants the GPU test's comparisons must catch."""
import numpy as np
import pytest

from oracle import ref64_surface as S
from oracle.ref64 import kernel

F = np.float32


def _grid_field(fn, lo, hi, s):
    o, dims = S.lattice(lo, hi, s)
    p = S.points(o, dims, s).astype(np.float64)
    return F(fn(p)).reshape(-1), o, dims


def _sphere(R, s, c=(0.013, -0.021, 0.007)):
    """phi = 2 - |p - c| / R (inside: |p - c| <= R), on the box [c - 2R, c + 2R]."""
    c = np.asarray(c)
    phi, o, dims = _grid_field(lambda p: 2.0 - np.linalg.norm(p - c, axis=1) / R, c - 2 * R, c + 2 * R, s)
    return S.polygonise(phi, o, dims, s, 1.0), phi, o, dims


def _single_particle(h=0.2, r=0.05, s=0.025, pad=True):
    x = np.array([[0.0113, -0.0071, 0.0029]], F)
    vol = F(0.8 * (2 * r) ** 3)
    lo, hi = S.default_box(x, h) if pad else (x.min(0), x.max(0))
    o, dims = S.lattice(lo, hi, s)
    phi64, _ = S.field64(x, vol, S.points(o, dims, s), h)
    iso = float(vol) * float(kernel(0, "w", np.array([0.5 * h]), h)[0][0])
    return x, vol, S.polygonise(F(phi64), o, dims, s, iso), phi64, o, dims, iso


def test_plane_gives_planar_vertices_exactly():
    """phi = 1.25 - z / 0.3: every vertex of the plane phi = 1 has the same float32 z, and z = 0.075 to rounding."""
    s = 0.01
    phi, o, dims = _grid_field(lambda p: 1.25 - p[:, 2] / 0.3, (-0.05, -0.04, 0.0), (0.05, 0.06, 0.15), s)
    v, t = S.polygonise(phi, o, dims, s, 1.0)
    assert len(t) and len(v)
    assert np.all(v[:, 2] == v[0, 2])
    assert abs(float(v[0, 2]) - 0.075) < 1e-6
    n = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    assert np.all(n[:, 2] > 0)  # counter-clockwise seen from outside: lower phi is +z


def test_sphere_volume_and_area_converge():
    R = 0.1
    err_v, err_a = [], []
    for s in (R / 3, R / 6, R / 12):
        (v, t), *_ = _sphere(R, s)
        assert S.watertight_oriented(t)
        assert S.components(len(v), t) == 1 and S.euler(len(v), t) == 2
        err_v.append(abs(S.volume(v, t) - 4 / 3 * np.pi * R ** 3) / (4 / 3 * np.pi * R ** 3))
        err_a.append(abs(S.area(v, t) - 4 * np.pi * R ** 2) / (4 * np.pi * R ** 2))
    assert err_v[0] > err_v[1] > err_v[2] and err_v[2] < 0.01
    assert err_a[2] < 0.05


def test_single_particle_one_closed_surface():
    _, _, (v, t), *_ = _single_particle()
    assert len(t) > 20
    assert S.watertight_oriented(t)
    assert S.components(len(v), t) == 1
    assert S.euler(len(v), t) == 2
    assert S.volume(v, t) > 0


def _cases(phi, dims, iso):
    nx, ny, nz = dims
    inside = (np.asarray(phi).reshape(nz, ny, nx) >= iso)
    seen = set()
    for tet in S.TETS:
        c = np.zeros((nz - 1, ny - 1, nx - 1), np.int64)
        for v, b in enumerate(tet):
            bx, by, bz = b & 1, (b >> 1) & 1, (b >> 2) & 1
            c |= inside[bz:nz - 1 + bz, by:ny - 1 + by, bx:nx - 1 + bx].astype(np.int64) << v
        seen |= set(np.unique(c).tolist())
    return seen


def test_random_field_exercises_all_16_cases_and_closes():
    rng = np.random.default_rng(7)
    dims = (14, 12, 10)
    phi = rng.random(dims[::-1]).astype(F)
    phi[0], phi[-1], phi[:, 0], phi[:, -1], phi[:, :, 0], phi[:, :, -1] = 0, 0, 0, 0, 0, 0
    assert _cases(phi, dims, 0.5) == set(range(16))
    v, t = S.polygonise(phi, np.zeros(3, F), np.array(dims), 0.1, 0.5)
    assert S.watertight_oriented(t)
    assert S.euler(len(v), t) % 2 == 0  # closed orientable surfaces (of any genus: the field is random)
    assert len(np.unique(t)) == len(v)  # every vertex is used


def test_field64_bound_covers_a_float32_sum():
    rng = np.random.default_rng(3)
    h, r = 0.2, 0.05
    x = rng.uniform(-0.2, 0.2, (300, 3)).astype(F)
    vol = F(0.8 * (2 * r) ** 3)
    o, dims = S.lattice(*S.default_box(x, h), 0.05)
    pts = S.points(o, dims, 0.05)
    phi64, b = S.field64(x, vol, pts, h)
    phi32 = np.zeros(len(pts), F)
    for j in range(len(x)):  # float32 sum in particle order
        d = (pts - x[j]).astype(F)
        rr = np.sqrt((d * d).sum(1, dtype=F)).astype(F)
        w = F(kernel(0, "w", rr.astype(np.float64), h)[0])
        phi32 = (phi32 + vol * w).astype(F)
    assert np.all(np.abs(phi32 - phi64) <= b)
    assert np.all(b <= 1e-2 * np.maximum(1.0, phi64))  # tight enough to see a wrong kernel or volume


# ---- mutants: each plausible bug is caught by the check that guards it ----------------------------------------------------
def test_mutant_split_other_diagonal():
    (v, t), phi, o, dims = _sphere(0.1, 0.1 / 6)
    nx, ny, nz = dims
    inside = phi.reshape(nz, ny, nx) >= 1.0
    mixed = inside[:-1, :-1, :-1] != inside[1:, 1:, 1:]  # cubes whose main diagonal the surface crosses
    kz, ky, kx = (int(a[len(a) // 2]) for a in np.nonzero(mixed))
    ti = kx + nx * (ky + ny * kz)
    vm, tm = S.polygonise(phi, o, dims, 0.1 / 6, 1.0, split=int(ti))
    assert not np.array_equal(tm, t)
    assert not S.watertight_oriented(tm)


@pytest.mark.parametrize("case", range(1, 15))
def test_mutant_flipped_case_winding(case):
    rng = np.random.default_rng(7)
    dims = (14, 12, 10)
    phi = rng.random(dims[::-1]).astype(F)
    phi[0], phi[-1], phi[:, 0], phi[:, -1], phi[:, :, 0], phi[:, :, -1] = 0, 0, 0, 0, 0, 0
    v, t = S.polygonise(phi, np.zeros(3, F), np.array(dims), 0.1, 0.5, flip_case=case)
    assert S.edge_counts(t)[0].min() == 2 and not S.watertight_oriented(t)  # still manifold, no longer oriented


def test_mutant_t_from_the_wrong_end():
    s = 0.01
    phi, o, dims = _grid_field(lambda p: 1.24 - p[:, 2] / 0.3, (-0.05, -0.04, 0.0), (0.05, 0.06, 0.15), s)
    v, _ = S.polygonise(phi, o, dims, s, 1.0)
    assert abs(float(v[0, 2]) - 0.072) < 1e-6
    vm, _ = S.polygonise(phi, o, dims, s, 1.0, t_from_outside=True)
    assert abs(float(vm[0, 2]) - 0.072) > 1e-3


def test_mutant_tie_rule_inverted():
    """Lattice values equal to iso: the mutant meshes a different surface, which the bit-exact comparison sees."""
    s = 0.01
    phi, o, dims = _grid_field(lambda p: 1.25 - np.round(p[:, 2] / s) * s / 0.2, (-0.03, -0.03, 0.0), (0.03, 0.03, 0.1), s)
    assert np.any(phi == F(1.0))
    v, t = S.polygonise(phi, o, dims, s, 1.0)
    vm, tm = S.polygonise(phi, o, dims, s, 1.0, tie_outside=True)
    assert not (np.array_equal(v, vm) and np.array_equal(t, tm))


def test_mutant_unaligned_origin():
    """Aligned lattices of two boxes share their points; origin = lo does not."""
    s = F(0.03)
    a, b = ((-0.101, 0.2, 0.05), (0.3, 0.5, 0.4)), ((-0.047, 0.23, 0.011), (0.35, 0.6, 0.5))
    oa, da = S.lattice(*a, s)
    ob, db = S.lattice(*b, s)
    ca, cb = S.coords(oa, da, s), S.coords(ob, db, s)
    assert all(np.intersect1d(ca[k], cb[k]).size >= 3 for k in range(3))
    ua, ub = S.coords(np.asarray(a[0], F), da, s), S.coords(np.asarray(b[0], F), db, s)
    assert not all(np.intersect1d(ua[k], ub[k]).size >= 3 for k in range(3))


def test_mutant_missing_h_pad():
    *_, (v, t), phi, o, dims, iso = _single_particle(pad=True)
    assert S.watertight_oriented(t)
    _, _, (vm, tm), *_ = _single_particle(pad=False)
    assert not (len(tm) and S.watertight_oriented(tm))


def test_mutant_normals_of_the_wrong_sign():
    x, vol, (v, t), *_ = _single_particle()
    n, m, gb = S.normals64(x, vol, v, 0.2)
    out = v.astype(np.float64) - x[0]
    assert np.all((n * out).sum(1) > 0)       # -grad phi points away from the particle
    assert np.all((-n * out).sum(1) < 0)      # the mutant's do not


def test_mutant_vertices_ordered_by_edge_first():
    (v, t), phi, o, dims = _sphere(0.1, 0.1 / 6)
    vm, tm = S.polygonise(phi, o, dims, 0.1 / 6, 1.0, edge_major=True)
    assert len(vm) == len(v) and not np.array_equal(vm, v)
