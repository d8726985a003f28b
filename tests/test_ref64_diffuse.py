"""The float64 diffuse-particle restatement (oracle/ref64_diffuse.py) against closed forms, and the mutants it must catch."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref64_diffuse as D  # noqa: E402

F = np.float32
H = 0.2
DESC = dict(ta_min=2.0, ta_max=8.0, wc_min=0.5, wc_max=4.0, k_min=0.1, k_max=2.0, k_ta=50.0, k_wc=50.0, lifetime=2.0, k_b=0.8,
            k_d=0.5, spray_below=6, bubble_above=20, capacity=1 << 20, seed=7, lo=[-np.inf] * 3, hi=[np.inf] * 3)


def _pot(x, v, n=None, mutant=None):
    x, v = np.asarray(x, F), np.asarray(v, F)
    n = np.zeros((len(x), 3)) if n is None else np.asarray(n, np.float64)
    return D.potentials64(x, v, F(1e-3), F(1000.0), n, np.zeros(len(x)), H, mutant=mutant)


@pytest.mark.parametrize("mutant", [None, "W"])
def test_trapped_air_of_two_particles(mutant):
    x = [[0.0, 0.0, 0.0], [0.1, 0.0, 0.0]]
    wt = 1.0 - float(F(0.1)) / H
    p = _pot(x, [[1.0, 0.0, 0.0], [-1.0, 0.0, 0.0]], mutant=mutant)          # approaching head-on: v^ . x^ = -1
    ok = np.allclose(p["ta"], 2.0 * 2.0 * wt, rtol=1e-12)
    assert ok == (mutant is None)
    p = _pot(x, [[-1.0, 0.0, 0.0], [1.0, 0.0, 0.0]])                          # separating: v^ . x^ = 1
    assert np.allclose(p["ta"], 0.0, atol=1e-15)
    p = _pot(x, [[1.0, 0.0, 0.0], [1.0, 0.0, 0.0]])                           # |v_ij| = 0
    assert np.all(p["ta"] == 0.0)


def _sheet(shape):
    """A layer of particles z = f(x, y) with upward normals, and the particle at the centre."""
    g = np.arange(-3, 4) * 0.05
    X, Y = np.meshgrid(g, g, indexing="ij")
    Z = {"flat": 0 * X, "crest": -2.0 * (X ** 2 + Y ** 2), "trough": 2.0 * (X ** 2 + Y ** 2)}[shape]
    x = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1).astype(F)
    grad = {"flat": (0 * X, 0 * Y), "crest": (-4.0 * X, -4.0 * Y), "trough": (4.0 * X, 4.0 * Y)}[shape]
    n = np.stack([-grad[0].ravel(), -grad[1].ravel(), np.ones(X.size)], 1)
    n /= np.linalg.norm(n, axis=1)[:, None]
    return x, n, int(np.argmin((x[:, :2] ** 2).sum(1)))


@pytest.mark.parametrize("mutant", [None, "convex"])
def test_wave_crest_on_sheet_crest_and_trough(mutant):
    v = np.tile([0.0, 0.0, 1.0], (49, 1))
    out = {}
    for shape in ("flat", "crest", "trough"):
        x, n, c = _sheet(shape)
        out[shape] = _pot(x, v, n, mutant)["kap"][c]
    assert out["flat"] == pytest.approx(0.0, abs=1e-12)
    if mutant is None:
        assert out["crest"] > 1e-3 and out["trough"] == pytest.approx(0.0, abs=1e-12)
    else:
        assert not (out["crest"] > 1e-3 and out["trough"] == pytest.approx(0.0, abs=1e-12))


@pytest.mark.parametrize("mutant", [None, "no_gate"])
def test_wave_crest_needs_the_velocity_along_the_normal(mutant):
    x, n, c = _sheet("crest")
    v = np.tile([1.0, 0.0, 0.0], (49, 1))                                      # v^ . n = 0 < 0.6 at the crest
    p = _pot(x, v, n, mutant)
    assert (p["wc"][c] == 0.0) == (mutant is None)
    assert p["kap"][c] > 0


def test_clamp_at_and_beyond_its_thresholds():
    I = np.array([-1.0, 2.0, 5.0, 8.0, 100.0])
    want = np.array([0.0, 0.0, 0.5, 1.0, 1.0])
    assert np.array_equal(D.phi(I, 2.0, 8.0), want)
    assert np.array_equal(D.phi32(I, 2.0, 8.0), want.astype(F))


@pytest.mark.parametrize("mutant", [None, "inclusive"])
def test_classification_thresholds_are_exclusive(mutant):
    xf = np.array([[0.02 * k, 0.0, 0.0] for k in range(1, 7)], F)            # exactly 6 fluid particles within h of the origin
    vf = np.zeros((6, 3), F)
    xd, vd = np.zeros((1, 3), F), np.zeros((1, 3), F)
    kinds = []
    for sb, ba in ((6, 20), (0, 6)):
        r = D.advect64(xd, vd, np.ones(1, F), xf, vf, H, dict(DESC, spray_below=sb, bubble_above=ba), 0.01, [0, -9.81, 0], mutant=mutant)
        assert r["nn"][0] == 6
        kinds.append(int(r["kind"][0]))
    assert (kinds == [D.FOAM, D.FOAM]) == (mutant is None)


def test_counts_round_stochastically():
    n = 200000
    ids = np.arange(n, dtype=np.uint32)
    e = np.full(n, 3.0, F)                                                     # Phi_k = 1
    for ta, want in ((5.0, 0.5 * 50 * 0.01), (8.0, 50 * 0.01)):
        c = D.counts32(np.full(n, ta, F), np.zeros(n, F), e, np.zeros(n), ids, DESC, 0.01, 3)
        assert abs(c.mean() - want) < 0.01 and set(np.unique(c)) <= {0, 1}
    c = D.counts32(np.full(4, 8.0, F), np.full(4, 4.0, F), np.full(4, 3.0, F), np.zeros(4), ids[:4], DESC, 1.0, 0)
    assert np.all(c == 100)                                                    # 50 + 50, + u < 1


@pytest.mark.parametrize("v", [[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1e-4, 0, -1], [0.3, -0.4, 0.5]])
def test_basis_is_orthonormal_and_samples_lie_in_their_cylinder(v):
    v = np.asarray(v, np.float64) * 2.0
    nv = v / np.linalg.norm(v)
    e1, e2 = D.basis(nv[None])
    M = np.stack([e1[0], e2[0], nv])
    assert np.allclose(M @ M.T, np.eye(3), atol=1e-12)
    xf, vf = np.zeros((1, 3), F), v[None].astype(F)
    x, vd, _, _, rows = D.emit64(xf, vf, [0], [5], [500], DESC, 0.02, 1, 0.05)
    o = vd - vf.astype(np.float64)
    assert np.all(np.linalg.norm(o, axis=1) <= 0.05 * (1 + 1e-12))
    assert np.allclose((o * nv).sum(1), 0.0, atol=1e-7)  # nv from the float64 v, the sample from its float32 copy
    along = ((x - o) * nv).sum(1)
    assert np.all(along >= -1e-7) and np.all(along <= np.linalg.norm(v) * 0.02 * (1 + 1e-6))


def test_emission_cut_at_capacity():
    xf, vf = np.zeros((3, 3), F), np.ones((3, 3), F)
    x, v, _, _, rows = D.emit64(xf, vf, [0, 0, 0], [1, 2, 3], [2, 3, 4], DESC, 0.01, 0, 0.05, room=4)
    assert rows.tolist() == [0, 0, 1, 1]
    x, v, _, _, rows = D.emit64(xf, vf, [0, 0, 0], [1, 2, 3], [2, 3, 4], DESC, 0.01, 0, 0.05, room=4, mutant="cut")
    assert len(rows) == 5  # the off-by-one the tests must catch


@pytest.mark.parametrize("mutant", [None, "all_age"])
def test_advection_of_each_kind(mutant):
    g = np.array([0.0, -9.81, 0.0])
    dt = 0.01
    # fluid: a dense cube of 27 particles moving at (1, 0, 0); diffuse: far away (spray), at the cube's corner (foam), at its centre
    c = (np.stack(np.meshgrid(*[np.arange(3) * 0.05] * 3, indexing="ij"), -1).reshape(-1, 3)).astype(F)
    vf = np.tile(F([1.0, 0.0, 0.0]), (27, 1))
    d = dict(DESC, spray_below=4, bubble_above=20)
    xd = np.array([[5.0, 5.0, 5.0], [0.17, 0.17, 0.17], [0.05, 0.05, 0.05]], F)
    vd = np.array([[0.0, 1.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]], F)
    r = D.advect64(xd, vd, np.full(3, 1.0, F), c, vf, H, d, dt, g, mutant=mutant)
    assert r["kind"].tolist() == [D.SPRAY, D.FOAM, D.BUBBLE], r["nn"]
    assert np.allclose(r["v"][0], [0.0, 1.0 - 0.0981, 0.0]) and np.allclose(r["x"][0], xd[0] + dt * r["v"][0])
    assert np.allclose(r["v"][1], [1.0, 0.0, 0.0]) and np.allclose(r["x"][1], xd[1] + dt * np.array([1.0, 0.0, 0.0]))
    assert np.allclose(r["v"][2], -dt * 0.8 * g + 0.5 * np.array([1.0, 0.0, 0.0]))
    ok = r["life"].tolist() == pytest.approx([1.0, 1.0 - dt, 1.0])
    assert ok == (mutant is None)


def test_the_hash_is_the_cpp_function(tmp_path):
    src = tmp_path / "h.cpp"
    src.write_text('#include <cstdio>\n#include "sph_hash.h"\nint main() {\n'
                   '  for (unsigned t = 0; t < 64; ++t) printf("%u %.9g\\n", sph_diffuse_hash(t * 2654435761u, t, t % 16, t * 977u, t % 5, t % 4),'
                   ' sph_hash_unit(sph_diffuse_hash(3, t, 1, t, 0, 0)));\n  return 0;\n}\n')
    exe = tmp_path / "h"
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "salva_b200", "csrc"), "-o", str(exe), str(src)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    t = np.arange(64, dtype=np.uint64)
    want = D.hash32((t * np.uint64(2654435761)) & D.M32, t, t % 16, (t * np.uint64(977)) & D.M32, t % 5, t % 4)
    wu = D.unit(D.hash32(3, t, 1, t, 0, 0))
    for k in range(64):
        a, b = lines[k].split()
        assert int(a) == int(want[k]) and F(b) == wu[k]
