"""The CFL-bounded substep rule of sph_world_set_substepping (DESIGN.md section 12) restated in float64, and the check the
GPU test applies to a substepped step.

TEST INFRASTRUCTURE ONLY.  Substep k of a step of length T starts with the remaining time R_k (R_0 = T, f32 on the host) and
computes, after the non-pressure forces,
    m   = max over the fluid particles of |v + a R_k|^2            (timestep_manager.rs:36-46)
    d   = (2 r) / sqrt(m) * cfl            (+inf when m == 0)
    n_k = clamp(ceil(R_k / d), max(1, min - k), max(1, max - k))  (a non-finite or NaN ratio takes the upper bound)
    dt_k = f32(R_k / n_k),  R_{k+1} = f32(R_k - dt_k)
and the step ends when R_{k+1} <= FLT_EPSILON.  `check` recomputes n_k in float64 from the v and a the substep saw and
compares it with the count the engine's dt_k implies; an R_k / d_k within `near` (relative) of an integer is reported
rather than compared, since the engine's float32 m may round it to either side.
"""
import math

import numpy as np

F = np.float32
FLT_EPS = float(np.finfo(np.float32).eps)


def max_sq(v, a, remaining):
    """m = max_i |v_i + a_i R|^2 in float64 (0 for no particles)."""
    v = np.asarray(v, np.float64).reshape(-1, 3)
    if len(v) == 0:
        return 0.0
    u = v + np.asarray(a, np.float64).reshape(-1, 3) * float(remaining)
    return float(np.max(np.sum(u * u, axis=1)))


def bound(m, r, cfl):
    """d = (2 r) / sqrt(m) * cfl; +inf for m == 0 (NaN for m = NaN, and for m = +inf with cfl = +inf)."""
    if m == 0.0:
        return math.inf
    with np.errstate(all="ignore"):
        return float(np.float64(2.0 * r) / np.sqrt(np.float64(m)) * np.float64(cfl))


def ratio(remaining, d):
    with np.errstate(all="ignore"):
        return float(np.float64(remaining) / np.float64(d))


def count(q, min_substeps, max_substeps, k):
    """n_k = clamp(ceil(q), max(1, min - k), max(1, max - k)); a non-finite q takes the upper bound."""
    lo, hi = max(1, min_substeps - k), max(1, max_substeps - k)
    if not math.isfinite(q):
        return hi
    return int(min(max(math.ceil(q), lo), hi))


def choose(v, a, remaining, r, cfl, min_substeps, max_substeps, k):
    """(n_k, d_k, R_k / d_k) of the substep that starts with `remaining` and sees velocities v and accelerations a."""
    d = bound(max_sq(v, a, remaining), r, cfl)
    q = ratio(remaining, d)
    return count(q, min_substeps, max_substeps, k), d, q


def split(T, state, r, cfl, min_substeps, max_substeps, rule=None):
    """The substep lengths of a step of length T.  state(k, dts_so_far) -> (v, a) is what substep k sees; rule (default
    `rule_reference`) turns (v, a, R_k, T, k) into dt_k.  The remaining time is kept in float32 as the engine keeps it."""
    rule = rule or rule_reference
    dts, R = [], F(T)
    while float(R) > FLT_EPS and len(dts) < 1000:
        v, a = state(len(dts), list(dts))
        dt = F(rule(v, a, R, F(T), len(dts), r, cfl, min_substeps, max_substeps))
        dts.append(dt)
        R = F(R - dt)
    return np.asarray(dts, F)


def rule_reference(v, a, R, T, k, r, cfl, mn, mx):
    n, _, _ = choose(v, a, R, r, cfl, mn, mx, k)
    return F(R) / F(n)


def check(T, dts, states, r, cfl, min_substeps, max_substeps, near=1e-5):
    """Check a step's substep lengths `dts` (float32, in order) against the rule.  states[k] = (v, a) that substep k saw.
    Returns dict(failures=[str], near=[k], n=[n_k implied by dts])."""
    dts = np.asarray(dts, F)
    out = dict(failures=[], near=[], n=[])
    fail = out["failures"].append
    if not min_substeps <= len(dts) <= max_substeps:
        fail("count %d outside [%d, %d]" % (len(dts), min_substeps, max_substeps))
    R = F(T)
    total = 0.0
    for k, dt in enumerate(dts):
        if not float(R) > FLT_EPS:
            fail("substep %d runs after the remaining time %g reached FLT_EPSILON" % (k, float(R)))
            break
        if not float(dt) > 0.0:
            fail("substep %d has length %g" % (k, float(dt)))
            break
        n_eng = int(round(float(R) / float(dt)))
        out["n"].append(n_eng)
        if n_eng < 1 or abs(float(dt) - float(R) / n_eng) > 2.0 ** -24 * float(R) / n_eng:
            fail("substep %d: dt %r is not R_k / n for an integer n (R_k = %r)" % (k, float(dt), float(R)))
        else:
            v, a = states[k]
            n_ref, d, q = choose(v, a, float(R), r, cfl, min_substeps, max_substeps, k)
            if math.isfinite(q) and q > 0 and abs(q - round(q)) <= near * q:
                out["near"].append(k)
            elif n_eng != n_ref:
                fail("substep %d: n = %d, the float64 rule gives %d (R_k / d_k = %r)" % (k, n_eng, n_ref, q))
            if n_ref < max(1, max_substeps - k) and not float(dt) <= d * (1.0 + 1e-6):
                fail("substep %d: dt %r exceeds the bound %r" % (k, float(dt), d))
        total += float(dt)
        R = F(R - dt)
    if float(R) > FLT_EPS:
        fail("the step ended with %g of its time left" % float(R))
    if abs(total - T) > 2.0 ** -23 * T * max(1, len(dts)):
        fail("the substeps add up to %r, not T = %r" % (total, T))
    return out
