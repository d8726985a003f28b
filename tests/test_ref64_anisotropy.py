"""The float64 restatement of the anisotropic surface kernels (oracle/ref64_anisotropy.py, DESIGN.md section 17): closed
forms, the float32 bounds against a float32 emulation, the mutants the device tests must catch, and the flatness the
kernels exist for.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref64_anisotropy as A  # noqa: E402
from oracle import ref64_surface as S  # noqa: E402

F = np.float32
R = 0.05
H = float(F(4 * R))
V0 = F(0.8 * (2 * R) ** 3)
ANI = dict(max_ratio=4.0, isolated_radius=0.5)  # stretched kernels: what the bounds and mutants exercise


def _lattice(nx, ny, nz, s=2 * R):
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3)
    return (g * s).astype(F)


def _rows(el, dtype=F):
    """The ellipsoids as device rows: centres and (e_k, a_k) per axis."""
    ax = np.concatenate([np.transpose(el["e"], (0, 2, 1)), el["a"][:, :, None]], axis=2)
    return el["centre"].astype(dtype), ax.astype(dtype)


def test_reduces_to_the_isotropic_field():
    p = _lattice(6, 5, 6) + np.random.default_rng(1).uniform(-0.3 * R, 0.3 * R, (180, 3)).astype(F)
    el = A.ellipsoids64(p, H, smoothing=0.0, max_ratio=1.0, isolated_radius=1.0)
    assert np.allclose(el["a"], H, rtol=0, atol=1e-12 * H)
    c, ax = _rows(el, np.float64)
    assert np.array_equal(c, p.astype(np.float64))
    o, dims = S.lattice(*S.default_box(p, H), R)
    pts = S.points(o, dims, R)
    phi, _ = A.field64(c, ax, V0, pts, H)
    ref, _ = S.field64(p, V0, pts, H)
    assert np.abs(phi - ref).max() <= 1e-12 * ref.max()


def test_interior_particle_of_a_cubic_lattice_is_a_ball():
    p = _lattice(7, 7, 7)
    el = A.ellipsoids64(p, H, **ANI)
    k = int(np.argmin(np.abs(p - p.mean(axis=0)).sum(axis=1)))
    s = el["sigma"][k]
    assert s[0] > 0 and (s[0] - s[2]) <= 1e-12 * s[0]
    assert np.allclose(el["centre"][k], p[k].astype(np.float64), atol=1e-12)
    assert np.allclose(el["a"][k], H, rtol=1e-12)


def test_top_face_particle_matches_the_lattice_sums():
    s = 2 * R
    p = _lattice(9, 5, 9, s)
    el = A.ellipsoids64(p, H, smoothing=0.9, **ANI)
    top = np.nonzero((p[:, 1] == p[:, 1].max()) & (np.abs(p[:, 0] - 4 * s) < 1e-6) & (np.abs(p[:, 2] - 4 * s) < 1e-6))[0][0]
    e3 = el["e"][top][:, 2]
    assert abs(abs(e3[1]) - 1.0) <= 1e-12
    # independent finite sums over the offsets (i, j, k) s with j <= 0 inside h, self weight 1
    w_, dy, dy2, dx2 = 0.0, 0.0, 0.0, 0.0
    n = int(H / s) + 1
    for i in range(-n, n + 1):
        for j in range(-n, 1):
            for k in range(-n, n + 1):
                off = np.array([i, j, k], F) * F(s)
                if (i, j, k) != (0, 0, 0):
                    d2 = F(F(off[0] * off[0] + off[1] * off[1]) + off[2] * off[2])
                    if not d2 <= F(H) * F(H):
                        continue
                r = float(np.sqrt((off.astype(np.float64) ** 2).sum()))
                wt = 1.0 - (r / H) ** 3
                w_ += wt
                dy += wt * float(off[1])
                dy2 += wt * float(off[1]) ** 2
                dx2 += wt * float(off[0]) ** 2
    my = dy / w_
    sy, sx = dy2 / w_ - my * my, dx2 / w_
    # the sums over exact multiples of s; the positions are those multiples rounded to float32
    assert abs((p[top, 1] - el["centre"][top][1]) - (-0.9 * my)) <= 1e-7
    assert abs(el["a"][top][2] / H - max(sy, sx / 4.0) / sx) <= 1e-6


def test_straight_line():
    p = np.zeros((30, 3), F)
    p[:, 0] = np.arange(30, dtype=F) * F(R)
    el = A.ellipsoids64(p, H, **ANI)
    mid = el["aniso"]
    assert mid.sum() > 10
    assert np.allclose(el["a"][mid][:, 1:], H / 4.0, rtol=1e-12)
    assert np.allclose(np.abs(el["e"][mid][:, 0, 0]), 1.0, atol=1e-12)


def test_small_neighbourhoods_switch_exactly_at_n_eps():
    # one particle with k neighbours at |x_ij|^2 = h^2 in float32 (on the axes, exact), plus one inside to make s1 > 0
    h32 = F(H)
    for k, expect in ((0, False), (5, False), (6, True)):
        dirs = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], F)
        nb = [np.array([F(0.5) * h32, 0, 0], F)] if k else []
        nb += list(dirs[: max(k - 1, 0)] * h32)
        p = np.concatenate([np.zeros((1, 3), F), np.asarray(nb, F).reshape(-1, 3)])
        el = A.ellipsoids64(p, H, min_neighbours=6, **ANI)
        assert el["N"][0] == k
        assert bool(el["aniso"][0]) == expect, k
        if not expect:
            assert np.allclose(el["a"][0], float(F(0.5 * H)))
    # a pair just past h is no neighbour
    q = np.array([[0, 0, 0], [np.nextafter(h32, F(1)), 0, 0]], F)
    assert A.ellipsoids64(q, H)["N"][0] == 0


def test_each_kernel_integrates_to_one():
    rng = np.random.default_rng(4)
    s = H / 24.0
    g = (np.arange(-24, 25) * s)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    pts = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    for _ in range(3):
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        a = np.sort(rng.uniform(H / 4, H, 3))[::-1]
        a[0] = H
        ax = np.concatenate([Q.T, a[:, None]], axis=1)[None].astype(np.float64)
        phi, _ = A.field64(np.zeros((1, 3)), ax, 1.0, pts, H)
        assert abs(phi.sum() * s ** 3 - 1.0) < 2e-3


def _random_neighbourhoods(seed):
    """Blocks, slabs, lines and near-degenerate clouds: near-equal eigenvalues and eigenvalues around s1 / k_r."""
    rng = np.random.default_rng(seed)
    out = [_lattice(6, 6, 6) + rng.uniform(-0.02 * R, 0.02 * R, (216, 3)).astype(F),
           _lattice(8, 2, 8) + rng.uniform(-0.4 * R, 0.4 * R, (128, 3)).astype(F)]
    for stretch in (1.0, 1.9, 2.0, 2.1, 4.0):  # the second axis at about 1 / stretch^2 of the first's variance
        c = rng.normal(size=(300, 3)) * np.array([H, H / stretch, H / 3.0]) * 0.6
        out.append((c + 1.0).astype(F))
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_bounds_cover_a_float32_evaluation(seed):
    for p in _random_neighbourhoods(seed):
        el = A.ellipsoids64(p, H, **ANI)
        c32, M32 = A.emulate32(p, H, **ANI)
        ce = np.abs(c32.astype(np.float64) - el["centre"])
        assert np.all(ce <= el["centre_bound"][:, None]), float((ce / el["centre_bound"][:, None]).max())
        me = np.sqrt(((M32 - el["M"]) ** 2).sum(axis=(1, 2)))
        ok = np.isfinite(el["M_bound"])
        assert ok.mean() > 0.9
        assert np.all(me[ok] <= el["M_bound"][ok]), float((me[ok] / el["M_bound"][ok]).max())
        # the bounds are tight enough to mean something: far below the size of what they bound
        assert np.median(el["M_bound"][ok]) < 5e-3 * H * H


MUTANTS = [dict(sqrt_radii=True), dict(clamp_before_sort=True), dict(weights_linear=True), dict(count_self=True),
           dict(swap_lambda=True)]


@pytest.mark.parametrize("mut", MUTANTS, ids=lambda m: next(iter(m)))
def test_ellipsoid_mutants_are_caught(mut):
    caught = False
    for p in _random_neighbourhoods(0)[:3] + [_edge_cloud()]:
        good = A.ellipsoids64(p, H, min_neighbours=6, **ANI)
        c32, M32 = A.emulate32(p, H, min_neighbours=6, **ANI)
        bad = A.ellipsoids64(p, H, min_neighbours=6, **ANI, **mut)
        dc = np.abs(bad["centre"] - c32) > good["centre_bound"][:, None]
        ok = np.isfinite(good["M_bound"])
        dm = np.sqrt(((bad["M"] - M32) ** 2).sum(axis=(1, 2)))[ok] > good["M_bound"][ok]
        caught |= bool(dc.any() or dm.any())
    assert caught


def _edge_cloud():
    """A particle with exactly N_eps neighbours: counting itself would not change it, but one with N_eps - 1 would."""
    h32 = F(H)
    nb = [np.array([F(0.5) * h32, 0, 0], F)] + [np.array(d, F) * h32 for d in ([-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1])]
    return np.concatenate([np.zeros((1, 3), F), np.asarray(nb, F)])


@pytest.mark.parametrize("mut", [dict(swap_G=True), dict(drop_det=True)], ids=lambda m: next(iter(m)))
def test_field_mutants_are_caught(mut):
    p = _lattice(8, 3, 8) + np.random.default_rng(2).uniform(-0.3 * R, 0.3 * R, (192, 3)).astype(F)
    c, ax = _rows(A.ellipsoids64(p, H, **ANI))
    o, dims = S.lattice(*S.default_box(p, H), R)
    pts = S.points(o, dims, R)
    phi, b = A.field64(c, ax, V0, pts, H)
    bad, _ = A.field64(c, ax, V0, pts, H, **mut)
    assert np.any(np.abs(bad - phi) > b)


def test_normal_mutant_is_caught():
    p = _lattice(8, 3, 8) + np.random.default_rng(2).uniform(-0.3 * R, 0.3 * R, (192, 3)).astype(F)
    c, ax = _rows(A.ellipsoids64(p, H, **ANI))
    v = (p[:50] + F(0.3 * H)).astype(F)
    n, m, gb = A.normals64(c, ax, V0, v, H)
    bad, _, _ = A.normals64(c, ax, V0, v, H, drop_G=True)
    ok = m > 1000 * gb
    assert ok.any()
    dev = np.linalg.norm(bad - n, axis=1)[ok]
    assert np.any(dev > (2.0 * np.sqrt(3.0) * gb / m)[ok] + 1e-5)


def flatness(p, aniso, spacing=R, iso=0.6):
    """(std of the heights of the top-face vertices, their count, mesh components) on the mesh of the float64 field: the
    vertices whose float64 normal lies within 10 degrees of +y and more than 2 h from the slab's sides.  aniso: None for
    the isotropic field, else the anisotropy parameters."""
    lo, hi = S.default_box(p, H)
    o, dims = S.lattice(lo, hi, spacing)
    pts = S.points(o, dims, spacing)
    if aniso is not None:
        c, ax = _rows(A.ellipsoids64(p, H, **aniso))
        phi, _ = A.field64(c, ax, V0, pts, H)
        verts, tris = S.polygonise(phi, o, dims, spacing, iso, dtype=np.float64)
        nrm, _, _ = A.normals64(c, ax, V0, verts, H)
    else:
        phi, _ = S.field64(p, V0, pts, H)
        verts, tris = S.polygonise(phi, o, dims, spacing, iso, dtype=np.float64)
        nrm, _, _ = S.normals64(p, V0, verts, H)
    pmin, pmax = p.min(axis=0), p.max(axis=0)
    sel = (nrm[:, 1] > np.cos(np.radians(10.0))) & (verts[:, 0] > pmin[0] + 2 * H) & (verts[:, 0] < pmax[0] - 2 * H) \
        & (verts[:, 2] > pmin[2] + 2 * H) & (verts[:, 2] < pmax[2] - 2 * H)
    return float(np.std(verts[sel, 1])), int(sel.sum()), S.components(len(verts), tris)


@pytest.mark.parametrize("layers", [4, 8])
def test_a_jittered_slab_is_flatter_with_the_default_anisotropy(layers):
    p = _lattice(20, layers, 20) + np.random.default_rng(7).uniform(-0.25 * R, 0.25 * R, (400 * layers, 3)).astype(F)
    iso, n_iso, c_iso = flatness(p, None)
    ani, n_ani, c_ani = flatness(p, {})
    print("top-face height std: isotropic %.3e (%d vertices), default anisotropy %.3e (%d), ratio %.3f" % (iso, n_iso, ani, n_ani, ani / iso))
    assert n_iso > 100 and n_ani > 100
    assert ani < iso
    assert c_iso == 1 and c_ani == 1  # no inner shells


def test_field_profile_of_stretched_kernels_through_a_lattice_slab():
    """Why k_r > 1 is not the default (DESIGN.md section 17): on an exact lattice only the outer layer is flattened (its
    longest axis held at h, a3 = 0.41 h), which concentrates its volume at the surface; the field one spacing under the
    surface falls from the isotropic 0.80 to 0.70, the margin that jittered fluid uses up."""
    p = _lattice(12, 8, 12)
    ys = np.arange(0.5, 0.8, 0.025)
    col = np.stack([np.full_like(ys, 0.6), ys, np.full_like(ys, 0.6)], 1).astype(F)
    iso, _ = S.field64(p, V0, col, H)
    el = A.ellipsoids64(p, H, **ANI)
    c, ax = _rows(el)
    ani, _ = A.field64(c, ax, V0, col, H)
    top = (np.abs(p[:, 0] - 0.6) < 1e-3) & (np.abs(p[:, 2] - 0.6) < 1e-3) & (p[:, 1] > 0.65)
    assert abs(el["a"][top][0, 2] / H - 0.41) < 0.01
    k = int(np.argmin(np.abs(ys - 0.6)))  # the second layer
    assert iso[k] > 0.79 and 0.68 < ani[k] < 0.72
