"""The float64 statement of the CFL substep rule (oracle/ref64_substeps.py) against closed forms, its four properties, and
the mutants the GPU test's comparison (ref64_substeps.check) must catch."""
import math

import numpy as np
import pytest

from oracle import ref64_substeps as S

F = np.float32
r = 0.025
G = np.array([0.0, -9.81, 0.0])


def _free_fall(v0, g=G):
    """A fluid in free fall: substep k sees v = v0 + g (time so far) and a = g for every particle."""
    v0 = np.asarray(v0, np.float64).reshape(-1, 3)

    def state(k, dts):
        t = float(np.sum(np.asarray(dts, np.float64)))
        return v0 + g * t, np.broadcast_to(g, v0.shape)
    return state


def _states(state, dts):
    return [state(k, list(dts[:k])) for k in range(len(dts))]


def test_a_uniform_velocity():
    """m = |v|^2, d = 2 r cfl / |v|: n = ceil(T |v| / (2 r cfl))."""
    v = np.tile([3.0, 0.0, 4.0], (7, 1))  # |v| = 5
    n, d, q = S.choose(v, np.zeros_like(v), 1 / 60, r, 0.4, 1, 10, 0)
    assert d == pytest.approx(2 * r * 0.4 / 5.0, rel=1e-15)
    assert q == pytest.approx((1 / 60) * 5.0 / (2 * r * 0.4), rel=1e-15)
    assert n == math.ceil(q) == 5


def test_gravity_only():
    """v = 0, a = g: m = (g R)^2."""
    R = 0.05
    m = S.max_sq(np.zeros((3, 3)), np.tile(G, (3, 1)), R)
    assert m == pytest.approx((9.81 * R) ** 2, rel=1e-15)
    n, d, _ = S.choose(np.zeros((3, 3)), np.tile(G, (3, 1)), R, r, 0.4, 1, 10, 0)
    assert d == pytest.approx(2 * r / (9.81 * R) * 0.4, rel=1e-15)
    assert n == math.ceil(R / d)


@pytest.mark.parametrize("N", [1, 2, 3, 7, 10])
def test_infinite_cfl_gives_exactly_n_equal_substeps(N):
    """(+inf, N, N): d = +inf, ceil(0) = 0 is lifted to the lower bound N - k, so every substep takes 1 / (N - k) of the rest."""
    T = 1 / 60
    dts = S.split(T, _free_fall(np.ones((4, 3))), r, math.inf, N, N)
    assert len(dts) == N
    assert np.allclose(dts, T / N, rtol=4e-7, atol=0)
    assert S.check(T, dts, _states(_free_fall(np.ones((4, 3))), dts), r, math.inf, N, N)["failures"] == []


def test_m_zero_is_an_infinite_bound():
    n, d, q = S.choose(np.zeros((5, 3)), np.zeros((5, 3)), 0.01, r, 0.4, 3, 10, 0)
    assert d == math.inf and q == 0.0 and n == 3
    assert S.count(S.ratio(0.01, S.bound(0.0, r, 0.4)), 1, 10, 0) == 1


def test_non_finite_ratios_take_the_upper_bound():
    assert S.count(math.inf, 1, 10, 2) == 8
    assert S.count(math.nan, 1, 10, 0) == 10
    assert S.choose(np.full((2, 3), np.inf), np.zeros((2, 3)), 0.01, r, 0.4, 1, 6, 1)[0] == 5


def test_min_binds_and_max_binds():
    slow = np.full((3, 3), 1e-3)
    assert S.choose(slow, np.zeros_like(slow), 1 / 60, r, 0.4, 4, 10, 0)[0] == 4
    assert S.choose(slow, np.zeros_like(slow), 1 / 60, r, 0.4, 4, 10, 2)[0] == 2
    fast = np.full((3, 3), 1e3)
    assert S.choose(fast, np.zeros_like(fast), 1 / 60, r, 0.4, 1, 10, 0)[0] == 10
    assert S.choose(fast, np.zeros_like(fast), 1 / 60, r, 0.4, 1, 10, 7)[0] == 3
    assert S.choose(fast, np.zeros_like(fast), 1 / 60, r, 0.4, 1, 10, 12)[0] == 1


CASES = [  # (v0 per particle, T, cfl, min, max)
    (np.array([[0.0, -2.0, 0.0], [0.5, 0.0, 0.0]]), 1 / 60, 0.4, 1, 10),
    (np.array([[1.0, -3.0, 0.5]]), 1 / 60, 0.4, 1, 10),
    (np.array([[0.0, -10.0, 0.0]]), 1 / 60, 0.4, 1, 4),
    (np.array([[0.0, 0.0, 0.0]]), 1 / 60, 0.4, 3, 10),
    (np.array([[0.0, -1.0, 0.0]]), 1 / 30, 0.25, 2, 6),
    (np.array([[4.0, 0.0, -4.0]]), 0.1, 1.0, 1, 64),
    (np.array([[0.0, 0.0, 0.0]]), 1e-6, 0.4, 1, 10),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_the_four_properties(case):
    """Every dt_k <= d_k unless max binds; sum dt_k = T up to f32 rounding; min <= count <= max; and the check passes."""
    v0, T, cfl, mn, mx = CASES[case]
    state = _free_fall(v0)
    dts = S.split(T, state, r, cfl, mn, mx)
    assert mn <= len(dts) <= mx
    assert abs(float(np.sum(dts.astype(np.float64))) - T) <= 2.0 ** -23 * T * len(dts)
    R = F(T)
    for k, dt in enumerate(dts):
        v, a = state(k, list(dts[:k]))
        n, d, _ = S.choose(v, a, float(R), r, cfl, mn, mx, k)
        if n < max(1, mx - k):
            assert float(dt) <= d * (1 + 1e-6)
        R = F(R - dt)
    res = S.check(T, dts, _states(state, dts), r, cfl, mn, mx)
    assert res["failures"] == [], res


def test_intermediate_counts_occur():
    """The scenes the mutants run on take more than one substep and fewer than max."""
    for v0, T, cfl, mn, mx in CASES[:2]:
        assert 1 < len(S.split(T, _free_fall(v0), r, cfl, mn, mx)) < mx


# ---- mutants ----------------------------------------------------------------------------------------------------------------
def _fixme_clamp(v, a, R, T, k, r, cfl, mn, mx):
    d = S.bound(S.max_sq(v, a, R), r, cfl)
    return min(max(d, float(T) / mx), float(T) / mn)   # compute_substep's commented-out rule: may overshoot T


def _t_for_r(v, a, R, T, k, r, cfl, mn, mx):
    n, _, _ = S.choose(v, a, float(T), r, cfl, mn, mx, k)
    return F(R) / F(n)


def _no_aR(v, a, R, T, k, r, cfl, mn, mx):
    n, _, _ = S.choose(v, np.zeros_like(np.asarray(v)), R, r, cfl, mn, mx, k)
    return F(R) / F(n)


def _r_for_2r(v, a, R, T, k, r, cfl, mn, mx):
    n, _, _ = S.choose(v, a, R, r / 2, cfl, mn, mx, k)
    return F(R) / F(n)


def _off_by_one(v, a, R, T, k, r, cfl, mn, mx):
    _, d, q = S.choose(v, a, R, r, cfl, mn, mx, k)
    return F(R) / F(S.count(math.ceil(q) + 1, mn, mx, k))


def _slivers(v, a, R, T, k, r, cfl, mn, mx):
    d = S.bound(S.max_sq(v, a, R), r, cfl)
    return min(d, float(R))   # steps of d, the last one capped at what is left


def _unreduced_bounds(v, a, R, T, k, r, cfl, mn, mx):
    n, _, _ = S.choose(v, a, R, r, cfl, mn, mx, 0)
    return F(R) / F(n)


MUTANTS = dict(fixme_clamp=_fixme_clamp, t_for_r=_t_for_r, no_aR=_no_aR, r_for_2r=_r_for_2r, off_by_one=_off_by_one,
               slivers=_slivers, unreduced_bounds=_unreduced_bounds)
MUTANT_CASES = dict(fixme_clamp=0, t_for_r=1, no_aR=1, r_for_2r=0, off_by_one=0, slivers=0, unreduced_bounds=2)


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_the_check_catches_the_mutant(name):
    """The mutant's substeps, run on the state they produce, fail ref64_substeps.check (the GPU test's comparison)."""
    v0, T, cfl, mn, mx = CASES[MUTANT_CASES[name]]
    if name == "unreduced_bounds":
        cfl, mn, mx = math.inf, 3, 3
    state = _free_fall(v0, G * 30 if name == "no_aR" else G)   # no_aR: an acceleration that dominates the velocity
    dts = S.split(T, state, r, cfl, mn, mx, rule=MUTANTS[name])
    ref = S.split(T, state, r, cfl, mn, mx)
    assert not np.array_equal(dts, ref), "the mutant does not change this scene's substeps"
    res = S.check(T, dts, _states(state, dts), r, cfl, mn, mx)
    assert res["failures"], (name, dts, res)
