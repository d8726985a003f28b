"""CPU checks of the cylinder and cone reference (oracle/ref64_revolution.py): the closed forms it reproduces, the float32
restatement of contact sampling (salva_b200.contact_sampling) within its bounds, and plausible bugs, each applied to the
reference, flagged."""
import numpy as np
import pytest

from oracle import ref64_colliders as C64
from oracle import ref64_revolution as RV
from oracle import ref64_sampling as RS
from salva_b200 import contact_sampling as CS

F = np.float32


def test_cylinder_vertical_rays_give_the_cap_pair():
    sh = RS.Shape(RV.CYLINDER, [0.3, 0.2])
    for cj, ck in ((0.0, 0.0), (0.1, -0.05), (-0.12, 0.15)):
        assert RV.crossings(sh, None, 1, F(cj), F(ck)) == ([(-float(F(0.3)), 0.0), (float(F(0.3)), 0.0)], np.inf)
    assert RV.crossings(sh, None, 1, F(0.2), F(0.1))[0] == []


@pytest.mark.parametrize("vol", [False, True])
def test_zero_height_cone_and_cylinder_give_the_same_keys(vol):
    a = RV.sample(RS.Shape(RV.CYLINDER, [0.0, 0.45]), 0.1, vol)
    b = RV.sample(RS.Shape(RV.CONE, [0.0, 0.45]), 0.1, vol)
    assert len(a.keys) > 0 or vol
    assert np.array_equal(a.keys, b.keys) and np.array_equal(a.undecided, b.undecided) and a.lines == b.lines


def test_zero_radius_cylinder_projects_as_a_zero_radius_capsule():
    pts = np.random.default_rng(1).uniform(-0.5, 0.5, (4000, 3)).astype(F)
    pts[:50, 0] = pts[:50, 2] = 0  # on the axis, inside and beyond the ends
    qc, ic, _ = CS.project_local(CS.CYLINDER, (0.3, 0.0), pts)
    qk, ik, _ = CS.project_local(CS.CAPSULE, (0.3, 0.0), pts)
    assert np.array_equal(qc, qk) and np.array_equal(ic, ik)
    P = RV.project64(RV.CYLINDER, 0.3, 0.0, pts.astype(np.float64), np.zeros(len(pts)))
    K = RV._capsule64(0.3, 0.0, pts.astype(np.float64), np.zeros(len(pts)))
    assert np.array_equal(P["q"], K["q"])


def test_distances_where_they_are_exactly_known():
    a, r, d = 0.25, 0.5, 0.125
    pts = np.array([[0, a + d, 0], [0, -a - d, 0], [r + d, 0, 0], [r + d, a + d, 0], [0, 0, 0]], np.float64)
    D = RV.project64(RV.CYLINDER, a, r, pts, np.zeros(len(pts)))["D"]
    assert np.allclose(D, [d, d, d, np.hypot(d, d), 0.0], rtol=0, atol=1e-15)
    cone = np.array([[0, a + d, 0], [0, -a - d, 0], [r + d, -a - d, 0], [r + d, -a, 0], [0, 0, 0]], np.float64)
    D = RV.project64(RV.CONE, a, r, cone, np.zeros(len(cone)))["D"]
    assert np.allclose(D, [d, d, np.hypot(d, d), d, 0.0], rtol=0, atol=1e-15)  # apex, base, below the rim, beside the rim
    # the float32 restatement agrees where the values are dyadic
    for kind, p, want in ((CS.CYLINDER, pts, [a, -a, 0.0]), (CS.CONE, cone, [a, -a, -a])):
        q, _, _ = CS.project_local(kind, (a, r), p[:3].astype(F))
        assert q[:, 1].tolist() == want


def test_degenerate_shapes_are_finite():
    pts = np.random.default_rng(2).uniform(-0.3, 0.3, (3000, 3)).astype(F)
    pts[:20] = 0
    for kind in (CS.CYLINDER, CS.CONE):
        for prm in ((0.0, 0.2), (0.2, 0.0), (0.0, 0.0)):
            q, inside, _ = CS.project_local(kind, prm, pts)
            assert np.all(np.isfinite(q)), (kind, prm)
            for vol in (False, True):
                RV.sample(RS.Shape(kind, prm), 0.05, vol)


def _steps(name, mutant=None, steps=None):
    sc = RV.SCENES[name]()
    pos = np.concatenate([f["positions"] for f in sc["fluids"]])
    vel = np.concatenate([f["velocities"] for f in sc["fluids"]])
    h = float(F(sc["radius"]) * F(2) * F(2))
    lag, worst, excluded, candidates, reasons = 0.0, {}, 0, 0, {}
    for k in range(steps or sc["steps"]):
        dt = C64.DTS[k % len(C64.DTS)]
        cols = C64.colliders_at(sc, k)
        p32, v32, s32 = CS.contact_sample(pos, vel, cols, lag, h, sc["radius"])
        res = RV.contact64(pos, vel, cols, lag, h, sc["radius"], mutant=mutant)
        for key, val in C64.check_restatement(res, p32, v32, s32).items():
            worst[key] = max(worst.get(key, 0.0), val)
        excluded += int(res.excluded.sum())
        candidates += res.candidates
        for key, n in res.reasons.items():
            reasons[key] = reasons.get(key, 0) + n
        pos, vel, lag = (p32 + v32 * F(dt)).astype(F), v32, dt
    return worst, excluded, candidates, reasons


@pytest.mark.parametrize("name", sorted(RV.SCENES))
def test_restatement_meets_the_float64_bounds(name):
    worst, excluded, candidates, reasons = _steps(name)
    print("\nREF64 revolution restatement %s worst %s excluded %d of %d %s" % (name, {k: round(v, 4) for k, v in worst.items()},
                                                                             excluded, candidates, reasons))
    assert max(worst.values()) <= 1.0, worst
    assert excluded <= 0.01 * candidates, (excluded, candidates, reasons)


@pytest.mark.parametrize("mutant", RV.CONTACT_MUTANTS)
def test_every_contact_mutant_is_flagged(mutant):
    worst, _, _, _ = _steps("posed", mutant, steps=3)
    assert max(worst.values()) > 1.0, (mutant, worst)


SAMPLE_CASES = {
    "apex_at_minus_a": (RS.Shape(RV.CONE, [0.5, 0.4]), 0.05, False),
    "axis_along_z": (RS.Shape(RV.CYLINDER, [0.5, 0.2]), 0.05, False),
    "radius_at_apex": (RS.Shape(RV.CONE, [0.5, 0.4]), 0.05, True),
    "open_caps": (RS.Shape(RV.CYLINDER, [0.3, 0.3]), 0.05, False),
    "rho2": (RS.Shape(RV.CONE, [0.5, 0.4]), 0.05, False),
}


@pytest.mark.parametrize("bug", RV.SAMPLE_BUGS)
def test_reference_flags_sampler_bug(bug):
    sh, r, vol = SAMPLE_CASES[bug]
    good = RV.sample(sh, r, vol)
    bad = RV.sample(sh, r, vol, bugs=[bug])
    missing, unexplained, _ = RS.compare(bad.keys, good)
    assert missing + unexplained > 0, bug


def test_sampling_undecided_fraction_is_small():
    for sh in (RS.Shape(RV.CYLINDER, [0.4, 0.3]), RS.Shape(RV.CONE, [0.4, 0.3])):
        for vol in (False, True):
            s = RV.sample(sh, 0.03, vol)
            assert len(s.keys) > 200 and len(s.undecided) + len(s.lines) < 0.05 * len(s.keys), (sh.kind, vol)


def query_points(kind, a, r, R, t, radius, n=20000, seed=5):
    """Points around a posed shape, dense near its surface and its AABB."""
    rng = np.random.default_rng(seed)
    ext = max(a, r) + 3 * radius
    loc = rng.uniform(-ext, ext, (n, 3))
    return (loc @ np.asarray(R, np.float64).T + t).astype(F)


@pytest.mark.parametrize("mutant", RV.QUERY_MUTANTS)
def test_every_query_mutant_is_flagged(mutant):
    """The |R| e box and a cone box centred on the translation visit cells the tight box does not, and a particle there
    within the radius is reported; a flipped cone reports other particles."""
    R = C64.rot(0.3, 0.7, 0.2).astype(np.float64)
    t = np.array([0.33, 0.41, 0.27])
    radius, h = 0.02, 0.08
    kind = RV.CYLINDER if mutant == "abs_r_box" else RV.CONE
    pts = query_points(kind, 0.2, 0.15, R, t, radius)
    hit, dec = RV.query64(kind, 0.2, 0.15, pts, R.astype(F), t.astype(F), h, radius)
    mh, md = RV.query64(kind, 0.2, 0.15, pts, R.astype(F), t.astype(F), h, radius, mutant=mutant)
    both = dec & md
    assert np.any(hit[both] != mh[both]), mutant
    assert (~dec).sum() < 0.02 * len(pts)
