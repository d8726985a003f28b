"""Float64 restatement of single DFSPH gather passes, each with the scale its float32 evaluation's error is measured against.

TEST INFRASTRUCTURE ONLY.  `numpy_ref.py` restates the whole step densely in float32; this module restates ONE pass at a time,
sparsely (contacts from a k-d tree, no grid, no lists), in float64 from the pass's own float32 inputs, so that a kernel's output
can be checked particle by particle against a bound that does not depend on the scene's largest value.

Contact membership is part of the definition, not of the precision: a pair is a contact exactly when the reference's float32
test (dx*dx + dy*dy) + dz*dz <= h*h, evaluated unfused, accepts it (contacts.rs:285).  Everything after that is float64.

Every pass returns a `Ref`: the float64 value and, per particle,
  A  the absolute evaluation: the pass's expression with every operand replaced by its absolute value and every
     subtraction by an addition (Higham's running-error quantity), the kernel value standing in as |W| or |W'/r|;
  K  the kernel term: sum over contacts of the kernel's own error scale `kerr` (see below) times the other operands;
  n  the summation depth (the number of terms a float32 evaluation accumulates).
`bound(ref, c_pass)` = (n + c_pass) u A + K with u = 2^-24.  The float32 sum of n terms whose values carry a relative error of
c_pass u each differs from the exact sum by at most (n - 1 + c_pass) u A to first order, whatever the summation order.

Kernel error scale.  A float32 kernel evaluation differs from the exact kernel at the exact distance in two ways:
  - its argument: r (or q = r / h) carries the roundings of the squared distance (dx, dx^2, two adds: <= 4u, i.e. <= 2u in r),
    of rsqrt.approx.ftz (PTX ISA: maximum relative error 2^-22.9 < 2.2u) and of r = d2 * inv_r and q = r * inv_h (1u each,
    inv_h 1u): |dr / r| <= 8u (the generic path's IEEE sqrt and divisions stay below that: <= 4.5u);
  - its polynomial: at most 8 roundings (the viscosity kernel's gradient, three quotients and two sums), each relative to
    the polynomial's absolute evaluation fa.
So kerr(r) = max over the two signs of |f(r (1 +- C_K u)) - f(r)| + C_K u fa(r) with C_K = 8.  The first part is the absolute
error of the kernel where (1 - q) cancels near q = 1, with no derivative involved, so it holds across the q = 1/2 seam and the
support's edge.  The kernels' normalisation constants (sigma: pi and h^3, 4.5u, dsigma6 two more; poly6: h^9 by repeated
products, 10.5u) are a relative error of every term and are counted in each pass's c_pass as C_NORM = 11.

Cites (reference src/): kernel/*.rs, solver/pressure/dfsph_solver.rs, solver/viscosity/xsph_viscosity.rs,
solver/surface_tension/akinci2013_surface_tension.rs, as restated in SURVEY.md Appendix A.
"""
from dataclasses import dataclass

import numpy as np
from scipy.spatial import cKDTree

F = np.float32
U = 2.0 ** -24
EPS32 = float(np.float32(1.1920929e-07))
C_K = 8
C_NORM = 11
MIN_NEIGHBORS = 20  # dfsph_solver.rs:62: no divergence solve below 20 contacts

# Per-pass c_pass: C_NORM plus the roundings of one term beyond its kernel value (dx: 1, v_i - v_j: 1, products and the sums
# of a dot product: 5, mass / pseudo-mass 1, inv_r of the gradient 1 + its own error 2.2 + d2's 2, the scale factor(s) 1-3).
C_PASS = dict(
    boundary_volume=C_NORM + 4,   # W (1) + 1 / sum (1) + 1 / vol read back as a sum (1) + margin 1
    density=C_NORM + 3,           # m_j or vol_b * rho0 (1), sigma * poly (1), fma (0) + margin 1
    alpha=C_NORM + 16,            # a = (g m) x: g 6.2, s 1, a 1 + dx 1, squares and sums of sq 3, 1 / den 1, margin 3
    divergence=C_NORM + 16,       # g 6.2, dv 1, dx 1, dot 5, dv * g 1, fma with m 0, pseudo-mass 1, margin 1
    predicted=C_NORM + 18,        # divergence + fma(d, dt, rho) 1 + margin 1
    update=C_NORM + 18,           # g 6.2, k_i + k_j 1, * m 1, * scale 1, * g 1, fma with x 1 + dx 1, v + vc 1, margin 4
    normals=C_NORM + 12,          # g 6.2, m / rho 1, * g 1, fma with x 1 + dx 1, * h 1, margin 1
    akinci=C_NORM + 16,           # cohesion 8 (r, powers, / r), -gamma m 1, cm x 2, n_i - n_j 1, sums 2, kij 2, margin 1
    xsph=C_NORM + 12,             # W 1, cf W 1, * m 1, / rho 1, v_j - v_i 1, fma 0, * inv_dt 1, acc + 1, margin 5
    # v_r = x . (v_i - v_j): dx 1, dv 1, dot 5; mu = h v_r / (d2 + 0.01 h^2): h v_r 1, d2 4, 0.01 h^2 2, + 1, / 1;
    # cs alpha mu - beta mu^2: 5; * cf 1; m_j / ((rho_i + rho_j) 0.5): 2 + / 1; * g (6.2) 1; fma with x 1; acc + 1; margin 2
    artificial=C_NORM + 36,
    # boundary forces, per boundary particle over its fluid contacts: pressure c = k_i vol_b rho0 inv_dt g (g 6.2, 4), then
    # c inv_dt m_i (2) and * dx (1 + 1), margin 2; adhesion: A(r) / r (r 2, / 1), * adh * vol_b * rho0 (3), * dx * m_i (2 + 1);
    # XSPH: c = cb W vol_b rho0 / rho_i (4), * (v_b - v_i) (1 + 1), * (-m_i inv_dt) (2), margin 2
    boundary_force=C_NORM + 16,
)


# ---- kernels: value f and absolute evaluation fa, both float64, for r >= 0 -------------------------------------------------
def _cubic(which, r, h):
    sigma = 8.0 / (np.pi * h ** 3)
    q = r / h
    inner, inside = q <= 0.5, q <= 1.0
    t = 1.0 - q
    if which == "w":
        f = np.where(inner, 1.0 + 6.0 * (q ** 3 - q ** 2), 2.0 * t ** 3)
        fa = np.where(inner, 1.0 + 6.0 * (q ** 3 + q ** 2), 2.0 * (1.0 + q) ** 3)
        return sigma * np.where(inside, f, 0.0), sigma * np.where(inside, fa, 0.0)
    rs = np.where(r > 0, r, 1.0)
    d6 = 6.0 * sigma / h
    f = np.where(inner, (3.0 * q - 2.0) * q, -t * t) * d6 / rs
    fa = np.where(inner, (3.0 * q + 2.0) * q, (1.0 + q) ** 2) * d6 / rs
    return np.where(inside & (q > 1e-5), f, 0.0), np.where(inside, fa, 0.0)


def _poly6(which, r, h):
    n = 315.0 / 64.0 / (np.pi * h ** 9)
    inside = r <= h
    if which == "w":
        return np.where(inside, n * (h * h - r * r) ** 3, 0.0), np.where(inside, n * (h * h + r * r) ** 3, 0.0)
    return np.where(inside, -6.0 * n * (h * h - r * r) ** 2, 0.0), np.where(inside, 6.0 * n * (h * h + r * r) ** 2, 0.0)


def _spiky(which, r, h):
    n = 15.0 / (np.pi * h ** 6)
    inside = r <= h
    if which == "w":
        return np.where(inside, n * (h - r) ** 3, 0.0), np.where(inside, n * (h + r) ** 3, 0.0)
    rs = np.where(r > 0, r, 1.0)
    return np.where(inside, -3.0 * n * (h - r) ** 2 / rs, 0.0), np.where(inside, 3.0 * n * (h + r) ** 2 / rs, 0.0)


def _viscosity(which, r, h):
    n = 15.0 / (2.0 * np.pi * h ** 3)
    inside = (r <= h) & (r > 0)
    rs = np.where(r > 0, r, 1.0)
    if which == "w":
        f = n * (rs * rs / (h * h) * (1.0 - rs / (2.0 * h)) + h / (2.0 * rs) - 1.0)
        fa = n * (rs * rs / (h * h) * (1.0 + rs / (2.0 * h)) + h / (2.0 * rs) + 1.0)
        return np.where(inside, f, 0.0), np.where(inside, fa, 0.0)
    f = n * (-3.0 * rs * rs / (2.0 * h ** 3) + 2.0 * rs / (h * h) - h / (2.0 * rs * rs)) / rs
    fa = n * (3.0 * rs * rs / (2.0 * h ** 3) + 2.0 * rs / (h * h) + h / (2.0 * rs * rs)) / rs
    return np.where(inside, f, 0.0), np.where(inside, fa, 0.0)


_KINDS = {0: _cubic, 1: _poly6, 2: _spiky, 3: _viscosity}


def kernel(kind, which, r, h):
    """(f, fa, kerr) of W (which = "w") or of g = W'(r) / r (which = "g"; grad W_ij = g x_ij) at the float64 distances r."""
    fn = _KINDS[kind]
    f, fa = fn(which, r, h)
    up, _ = fn(which, r * (1.0 + C_K * U), h)
    dn, _ = fn(which, r * (1.0 - C_K * U), h)
    kerr = np.maximum(np.abs(up - f), np.abs(dn - f)) + C_K * U * fa
    return f, fa, kerr


def grad_threshold(kind, h):
    """Squared distance at or below which the gradient is zero: |x|^2 <= eps^2 (kernel.rs:18-24), and for the cubic spline
    also q <= 1e-5 (cubic_spline_kernel.rs:64); the float32 threshold the kernels compare against."""
    a = EPS32 * EPS32
    return float(F(max(a, (1e-5 * h) ** 2))) if kind == 0 else a


# ---- contacts --------------------------------------------------------------------------------------------------------------
@dataclass
class Pairs:
    """Contacts as flat arrays, grouped by i: x = x_i - x_j in float64 (exact: the difference of two float32 values)."""
    i: np.ndarray
    j: np.ndarray
    x: np.ndarray

    def __post_init__(self):
        self.d2 = (self.x * self.x).sum(axis=1)
        self.r = np.sqrt(self.d2)

    def subset(self, keep):
        return Pairs(self.i[keep], self.j[keep], self.x[keep])

    def rank(self):
        """Position of every contact in its particle's list, in this order (0, 1, ... per i)."""
        start = np.searchsorted(self.i, self.i, side="left")
        return np.arange(len(self.i)) - start


def f32_d2(a, b):
    """The reference's float32 squared distance, unfused: (dx*dx + dy*dy) + dz*dz."""
    d = (a - b).astype(F)
    return ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F)


def _round_f32(fr):
    """The float32 nearest to the exact rational fr, ties to even."""
    from fractions import Fraction
    c = F(float(fr))
    cands = [np.nextafter(c, F(-np.inf)), c, np.nextafter(c, F(np.inf))]
    return min(cands, key=lambda x: (abs(Fraction(float(x)) - fr), int(np.array(x, F).view(np.uint32)) & 1))


def fma_d2(a, b):
    """d2 as the CUDA pair evaluation forms it, fma(dz, dz, fma(dy, dy, dx * dx)), emulated exactly: products of float32
    values are exact rationals, and each fma rounds its exact result once."""
    from fractions import Fraction
    d = (a - b).astype(F)
    out = np.empty(len(d), F)
    for k, (x, y, z) in enumerate(d.tolist()):
        p = F(F(x) * F(x))
        s = _round_f32(Fraction(y) * Fraction(y) + Fraction(float(p)))
        out[k] = _round_f32(Fraction(z) * Fraction(z) + Fraction(float(s)))
    return out


def contacts(P, Q, h, allowed, same=False):
    """Contacts of every point of P (float32) with the points of Q: the f32 test on k-d tree candidates within h (1 + 1e-5).
    allowed(i, j) -> bool mask (interaction groups).  same: Q is P (self contacts included, as the reference lists them)."""
    h32 = F(h)
    h2 = F(h32 * h32)
    tp = cKDTree(P.astype(np.float64))
    reach = float(h32) * (1.0 + 1e-5)
    if same:
        ij = tp.query_pairs(reach, output_type="ndarray")
        i = np.concatenate([ij[:, 0], ij[:, 1], np.arange(len(P))])
        j = np.concatenate([ij[:, 1], ij[:, 0], np.arange(len(P))])
    elif len(Q):
        m = tp.sparse_distance_matrix(cKDTree(Q.astype(np.float64)), reach, output_type="ndarray")
        i, j = m["i"].astype(np.int64), m["j"].astype(np.int64)
        # sparse_distance_matrix drops exact zero distances: coincident points are contacts too
        zi, zj = _coincident(P, Q)
        i, j = np.concatenate([i, zi]), np.concatenate([j, zj])
    else:
        i = j = np.zeros(0, np.int64)
    keep = f32_d2(P[i], Q[j]) <= h2
    keep &= allowed(i, j)
    i, j = i[keep], j[keep]
    o = np.lexsort((j, i))
    i, j = i[o], j[o]
    return Pairs(i, j, P[i].astype(np.float64) - Q[j].astype(np.float64))


def _coincident(P, Q):
    key = {}
    for k, q in enumerate(Q.tolist()):
        key.setdefault(tuple(q), []).append(k)
    hits = [(k, j) for k, p in enumerate(P.tolist()) for j in key.get(tuple(p), ())]
    if not hits:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    a = np.array(hits, np.int64)
    return a[:, 0], a[:, 1]


# ---- results ---------------------------------------------------------------------------------------------------------------
@dataclass
class Ref:
    value: np.ndarray
    A: np.ndarray
    K: np.ndarray
    n: np.ndarray

    def bound(self, c_pass):
        n = self.n if self.value.ndim == 1 else self.n[:, None]
        return (n + c_pass) * U * self.A + self.K


def _sum(n, idx, vals):
    if vals.ndim == 1:
        return np.bincount(idx, vals, n)
    return np.stack([np.bincount(idx, vals[:, c], n) for c in range(vals.shape[1])], axis=1)


def ratio(gpu, ref, c_pass):
    """|gpu - ref| / bound per particle (and component); 0 where both are exact, inf where the bound is 0 and they differ."""
    err = np.abs(np.asarray(gpu, np.float64) - ref.value)
    b = ref.bound(c_pass)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, np.inf))
    return r


# ---- passes ----------------------------------------------------------------------------------------------------------------
class Passes:
    """The float64 passes of one scene.  P: fluid positions (float32, all fluids concatenated), fid: fluid of each particle,
    rho0: per-particle rest density (float32), mass: per-particle mass (float32, vol * rho0 as the engine forms it),
    BP / bid: boundary positions and boundary of each, allowed_ff / allowed_fb: interaction-group masks over (i, j)."""

    def __init__(self, h, P, fid, rho0, mass, BP, bid, allowed_ff=None, allowed_fb=None, allowed_bb=None, kw=0, kg=0):
        self.h = float(F(h))
        self.P, self.fid = P, fid
        self.rho0 = np.asarray(rho0, F).astype(np.float64)
        self.mass = np.asarray(mass, F).astype(np.float64)
        self.BP, self.bid = BP, bid
        self.kw, self.kg = kw, kg
        self.N = len(P)
        every = lambda i, j: np.ones(len(i), bool)  # noqa: E731
        self.ff = contacts(P, P, self.h, allowed_ff or every, same=True)
        self.fb = contacts(P, BP, self.h, allowed_fb or every)
        self.bb = contacts(BP, BP, self.h, allowed_bb or every, same=True)
        self.nf = np.bincount(self.ff.i, minlength=self.N)
        self.nb = np.bincount(self.fb.i, minlength=self.N)

    # ambiguous float decisions: the gradient's zero threshold
    def ambiguous(self, pairs=None):
        """Particles with a contact whose squared distance lies within the float32 d2's rounding of the gradient's zero
        threshold: there the kernel may take either side."""
        t = grad_threshold(self.kg, self.h)
        out = np.zeros(self.N, bool)
        for pr in ([self.ff, self.fb] if pairs is None else pairs):
            near = np.abs(pr.d2 - t) <= 8 * U * t
            out[pr.i[near]] = True
        return out

    def _g(self, pr):
        g, ga, ge = kernel(self.kg, "g", pr.r, self.h)
        z = pr.d2 <= grad_threshold(self.kg, self.h)
        return np.where(z, 0.0, g), np.where(z, 0.0, ga), np.where(z, 0.0, ge)

    def _w(self, pr):
        return kernel(self.kw, "w", pr.r, self.h)

    def boundary_volume_sum(self):
        """sum_b' W(x_b - x_b') over the boundary's own contacts; the boundary volume is its reciprocal."""
        w, _, we = self._w(self.bb)
        nb = len(self.BP)
        return Ref(_sum(nb, self.bb.i, w), _sum(nb, self.bb.i, np.abs(w)), _sum(nb, self.bb.i, we),
                   np.bincount(self.bb.i, minlength=nb).astype(np.float64))

    def density(self, bvol, rho0_b=None, ff=None, fb=None):
        """rho_i = sum_j m_j W_ij + sum_b vol_b rho0_i W_ib (dfsph_solver.rs:628-665).  bvol: the engine's float32 volumes."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho0_b = self.rho0 if rho0_b is None else rho0_b
        w, _, we = self._w(ff)
        m = self.mass[ff.j]
        wb, _, wbe = self._w(fb)
        mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * rho0_b[fb.i]
        N = self.N
        val = _sum(N, ff.i, m * w) + _sum(N, fb.i, mb * wb)
        A = _sum(N, ff.i, np.abs(m * w)) + _sum(N, fb.i, np.abs(mb * wb))
        K = _sum(N, ff.i, np.abs(m) * we) + _sum(N, fb.i, np.abs(mb) * wbe)
        return Ref(val, A, K, (self._n(ff) + self._n(fb)).astype(np.float64))

    def _n(self, pr):
        return np.bincount(pr.i, minlength=self.N)

    def _grad_terms(self, pr, weight, weight_abs=None):
        """a = weight g x (a vector per contact), its absolute evaluation and its kernel part."""
        g, _, ge = self._g(pr)
        wa = np.abs(weight) if weight_abs is None else weight_abs
        a = (weight * g)[:, None] * pr.x
        aA = (wa * np.abs(g))[:, None] * np.abs(pr.x)
        aK = (wa * ge)[:, None] * np.abs(pr.x)
        return a, aA, aK

    def den(self, bvol, rho0_b=None):
        """alpha's denominator sum_j |m_j grad W_ij|^2 + |sum_j m_j grad W_ij|^2 (boundaries with vol_b rho0_i) and its error
        bound, propagated explicitly: the sum of gradients cancels in the interior, so its square is bounded from the
        errors of its components."""
        rho0_b = self.rho0 if rho0_b is None else rho0_b
        N = self.N
        mb = np.asarray(bvol, F).astype(np.float64)[self.fb.j] * rho0_b[self.fb.i]
        parts = [self._grad_terms(self.ff, self.mass[self.ff.j]), self._grad_terms(self.fb, mb)]
        idx = [self.ff.i, self.fb.i]
        n = (self.nf + self.nb).astype(np.float64)
        c = C_PASS["alpha"]
        sq = sum(_sum(N, ix, (a * a).sum(1)) for (a, _, _), ix in zip(parts, idx))
        gs = sum(_sum(N, ix, a) for (a, _, _), ix in zip(parts, idx))
        # per-term errors of a: c u |a| + kernel part
        ea = [(c * U * aA + aK) for (_, aA, aK) in parts]
        e_gs = sum(_sum(N, ix, aA) for (_, aA, _), ix in zip(parts, idx)) * (n * U)[:, None] + \
            sum(_sum(N, ix, e) for e, ix in zip(ea, idx))
        sqA = sum(_sum(N, ix, (aA * aA).sum(1)) for (_, aA, _), ix in zip(parts, idx))
        e_sq = (n + 3) * U * sqA + sum(_sum(N, ix, (2 * aA * e + e * e).sum(1)) for (_, aA, _), e, ix in zip(parts, ea, idx))
        gsA = np.abs(gs)
        e_den = e_sq + (2 * gsA * e_gs + e_gs * e_gs).sum(1) + 4 * U * ((gs * gs).sum(1) + sq)
        val = sq + (gs * gs).sum(1)
        return Ref(val, np.zeros(N), e_den + 2 * U * val, n)

    def divergence(self, vs, bvol, predicted=False, bvel=None, dens=None, dt=0.0, gate=True, rho0_b=None, ff=None, fb=None,
                   vj=None, min_neighbors=MIN_NEIGHBORS):
        """sum_j m_j (v*_i - v*_j) . grad W_ij + sum_b vol_b rho0_i (v*_i [- v_b]) . grad W_ib.
        Evaluation (predicted = False): 0 below `min_neighbors` contacts, then max(., 0) (dfsph_solver.rs:279-356).
        Predicted density: rho_i + dt * (the sum with boundary velocities), no gate (dfsph_solver.rs:98-162).
        vj: per-contact neighbour velocities (default vs[j])."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho0_b = self.rho0 if rho0_b is None else rho0_b
        N = self.N
        vs = np.asarray(vs, F).astype(np.float64)
        g, _, ge = self._g(ff)
        m = self.mass[ff.j]
        dv = vs[ff.i] - (vs[ff.j] if vj is None else np.asarray(vj, F).astype(np.float64))
        t = m * g * (dv * ff.x).sum(1)
        tA = np.abs(m * g) * (np.abs(dv) * np.abs(ff.x)).sum(1)
        tK = np.abs(m) * ge * (np.abs(dv) * np.abs(ff.x)).sum(1)
        gb, _, gbe = self._g(fb)
        mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * rho0_b[fb.i]
        dvb = vs[fb.i] - (np.asarray(bvel, F).astype(np.float64)[fb.j] if predicted else 0.0)
        tb = mb * gb * (dvb * fb.x).sum(1)
        tbA = np.abs(mb * gb) * (np.abs(dvb) * np.abs(fb.x)).sum(1)
        tbK = np.abs(mb) * gbe * (np.abs(dvb) * np.abs(fb.x)).sum(1)
        val = _sum(N, ff.i, t) + _sum(N, fb.i, tb)
        A = _sum(N, ff.i, tA) + _sum(N, fb.i, tbA)
        K = _sum(N, ff.i, tK) + _sum(N, fb.i, tbK)
        n = (self._n(ff) + self._n(fb)).astype(np.float64)
        if predicted:
            d = np.asarray(dens, F).astype(np.float64)
            dt = float(F(dt))
            return Ref(d + dt * val, np.abs(d) + dt * A, dt * K, n + 1)
        if gate:
            off = (self.nf + self.nb) < min_neighbors   # the gate counts the full lists
            val, A, K = np.where(off, 0.0, val), np.where(off, 0.0, A), np.where(off, 0.0, K)
        return Ref(np.maximum(val, 0.0), A, K, n)   # max(., 0) is 1-Lipschitz: the bound carries over

    def update(self, kappa, bvol, v0, pressure=False, inv_dt=0.0, rho0_b=None, kappa_b=None, ff=None, fb=None):
        """v0 - [sum_j (k_i + k_j) m_j grad W_ij + sum_b k_i vol_b rho0_i grad W_ib] * scale (dfsph_solver.rs:218-277, 358-409).
        pressure: scale = inv_dt and the boundary term only where k_i > 0; else scale = 1.  kappa: the float32 kappas the
        kernels read; kappa_b: the k_i of the boundary term (default kappa)."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho0_b = self.rho0 if rho0_b is None else rho0_b
        N = self.N
        k = np.asarray(kappa, F).astype(np.float64)
        kb = k if kappa_b is None else np.asarray(kappa_b, F).astype(np.float64)
        s = float(F(inv_dt)) if pressure else 1.0
        a, aA, aK = self._grad_terms(ff, (k[ff.i] + k[ff.j]) * self.mass[ff.j] * s,
                                     (np.abs(k[ff.i]) + np.abs(k[ff.j])) * self.mass[ff.j] * s)
        mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * rho0_b[fb.i]
        bw = kb[fb.i] * mb * s
        if pressure and kappa_b is None:
            bw = np.where(kb[fb.i] > 0, bw, 0.0)
        b, bA, bK = self._grad_terms(fb, bw)
        v0 = np.asarray(v0, F).astype(np.float64)
        val = v0 - _sum(N, ff.i, a) - _sum(N, fb.i, b)
        A = np.abs(v0) + _sum(N, ff.i, aA) + _sum(N, fb.i, bA)
        K = _sum(N, ff.i, aK) + _sum(N, fb.i, bK)
        return Ref(val, A, K, (self._n(ff) + self._n(fb) + 1).astype(np.float64))

    def akinci(self, dens, gamma, adhesion, bvol, rho_j=None, ff=None, fb=None):
        """Akinci2013SurfaceTension (akinci2013_surface_tension.rs:43-192): normals n_i = h sum_j (m_j / rho_j) grad W_ij over
        the same fluid, then the fluid force sum_j kij (-gamma (n_i - n_j) - gamma m_j C(r) x_ij / r), kij = 2 rho0 /
        (rho_i + rho_j), and the adhesion -adh vol_b rho0 A(r) x_ib / r.  rho_j: per-contact neighbour densities of the
        normals (default dens[j]).  The normals' own error bound is carried into the force's bound."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        N, h = self.N, self.h
        same = self.fid[ff.i] == self.fid[ff.j]
        sf = ff.subset(same)
        rho = np.asarray(dens, F).astype(np.float64)
        rj = rho[sf.j] if rho_j is None else np.asarray(rho_j, F).astype(np.float64)[same]
        a, aA, aK = self._grad_terms(sf, self.mass[sf.j] / rj)
        nrm = h * _sum(N, sf.i, a)
        nn = self._n(sf).astype(np.float64)
        e_n = h * ((nn + C_PASS["normals"])[:, None] * U * _sum(N, sf.i, aA) + _sum(N, sf.i, aK))
        gamma = float(F(gamma))
        r = np.where(sf.r > 0, sf.r, 1.0)
        coh, coha, cohe = _cohesion(sf.r, h)
        ok = sf.d2 > EPS32 * EPS32
        cm = np.where(ok, -gamma * self.mass[sf.j] * coh / r, 0.0)
        cmA = np.where(ok, abs(gamma) * self.mass[sf.j] * coha / r, 0.0)
        cmK = np.where(ok, abs(gamma) * self.mass[sf.j] * cohe / r, 0.0)
        kij = 2.0 * self.rho0[sf.i] / (rho[sf.i] + rho[sf.j])
        dn = nrm[sf.i] - nrm[sf.j]
        t = kij[:, None] * (-gamma * dn + cm[:, None] * sf.x)
        tA = kij[:, None] * (abs(gamma) * (np.abs(nrm[sf.i]) + np.abs(nrm[sf.j])) + cmA[:, None] * np.abs(sf.x))
        tK = kij[:, None] * (cmK[:, None] * np.abs(sf.x) + abs(gamma) * (e_n[sf.i] + e_n[sf.j]))
        val, A, K = _sum(N, sf.i, t), _sum(N, sf.i, tA), _sum(N, sf.i, tK)
        n = nn.copy()
        if adhesion != 0:
            adh = float(F(adhesion))
            rb = np.where(fb.r > 0, fb.r, 1.0)
            ad, ada, ade = _adhesion(fb.r, h)
            okb = fb.d2 > EPS32 * EPS32
            mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * self.rho0[fb.i]
            c = np.where(okb, adh * mb * ad / rb, 0.0)
            val -= _sum(N, fb.i, c[:, None] * fb.x)
            A += _sum(N, fb.i, np.where(okb, abs(adh) * mb * ada / rb, 0.0)[:, None] * np.abs(fb.x))
            K += _sum(N, fb.i, np.where(okb, abs(adh) * mb * ade / rb, 0.0)[:, None] * np.abs(fb.x))
            n += self._n(fb)
        return Ref(val, A, K, n)

    def _on_boundary(self, pr, t, tA, tK):
        """Per-contact vectors of fluid-boundary contacts summed onto the boundary particles (Boundary::apply_force)."""
        nb = len(self.BP)
        return Ref(_sum(nb, pr.j, t), _sum(nb, pr.j, tA), _sum(nb, pr.j, tK), np.bincount(pr.j, minlength=nb).astype(np.float64))

    def pressure_boundary_force(self, kappa, bvol, inv_dt, scale_m_inv_dt=True):
        """The force a pressure update puts on boundary particles (dfsph_solver.rs:267-272): for every contact with
        k_i > 0, (k_i vol_b rho0_i inv_dt g_ib) inv_dt m_i x_ib.  scale_m_inv_dt = False drops the second inv_dt m_i."""
        fb = self.fb
        k = np.asarray(kappa, F).astype(np.float64)[fb.i]
        s = float(F(inv_dt))
        mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * self.rho0[fb.i]
        w = np.where(k > 0, k * mb * s, 0.0) * ((s * self.mass[fb.i]) if scale_m_inv_dt else 1.0)
        return self._on_boundary(fb, *self._grad_terms(fb, w))

    def adhesion_boundary_force(self, adhesion, bvol):
        """Akinci2013's adhesion on boundary particles (akinci2013_surface_tension.rs:188): adh vol_b rho0_i A(r) / r x_ib m_i."""
        fb = self.fb
        rb = np.where(fb.r > 0, fb.r, 1.0)
        ad, ada, ade = _adhesion(fb.r, self.h)
        ok = fb.d2 > EPS32 * EPS32
        c = abs(float(F(adhesion))) * np.asarray(bvol, F).astype(np.float64)[fb.j] * self.rho0[fb.i] * self.mass[fb.i] / rb
        sgn = np.sign(float(F(adhesion)))
        t = np.where(ok, sgn * c * ad, 0.0)[:, None] * fb.x
        tA = np.where(ok, c * ada, 0.0)[:, None] * np.abs(fb.x)
        tK = np.where(ok, c * ade, 0.0)[:, None] * np.abs(fb.x)
        return self._on_boundary(fb, t, tA, tK)

    def xsph_boundary_force(self, vel, dens, cb, inv_dt, bvel, bvol):
        """XSPH's boundary term on boundary particles (xsph_viscosity.rs:87-88): -m_i inv_dt cb W vol_b rho0_i / rho_i (v_b - v_i)."""
        fb = self.fb
        v = np.asarray(vel, F).astype(np.float64)
        rho = np.asarray(dens, F).astype(np.float64)
        wb, _, wbe = self._w(fb)
        c = -self.mass[fb.i] * float(F(inv_dt)) * float(F(cb)) * np.asarray(bvol, F).astype(np.float64)[fb.j] * self.rho0[fb.i] / rho[fb.i]
        dvb = np.asarray(bvel, F).astype(np.float64)[fb.j] - v[fb.i]
        return self._on_boundary(fb, (c * wb)[:, None] * dvb, np.abs(c * wb)[:, None] * np.abs(dvb), (np.abs(c) * wbe)[:, None] * np.abs(dvb))

    def artificial(self, vel, dens, cf, cb, alpha, beta, cs, bvel, bvol, vr_gate=True):
        """ArtificialViscosity (artificial_viscosity.rs:40-124): over contacts of the same fluid with v_r = x_ij . (v_i - v_j)
        < 0, mu = h v_r / (|x_ij|^2 + 0.01 h^2) and cf (cs alpha mu - beta mu^2) m_j / ((rho_i + rho_j) / 2) grad W_ij; the
        boundary term likewise with cb, v_b and vol_b rho0_i / rho_i.  Returns (Ref, ambiguous): particles with a contact whose
        v_r is within its rounding of 0 (the kernel may take either side) are marked.  vr_gate = False drops the v_r < 0
        condition."""
        N, h = self.N, self.h
        v = np.asarray(vel, F).astype(np.float64)
        rho = np.asarray(dens, F).astype(np.float64)
        al, be, c_s = float(F(alpha)), float(F(beta)), float(F(cs))
        eta2 = float(F(F(F(h) * F(h)) * F(0.01)))
        amb = np.zeros(N, bool)
        val, A, K, n = np.zeros((N, 3)), np.zeros((N, 3)), np.zeros((N, 3)), np.zeros(N)
        sf = self.ff.subset(self.fid[self.ff.i] == self.fid[self.ff.j])
        for pr, coef, vj, scale in (
                (sf, float(F(cf)), lambda pr: v[pr.j], lambda pr: self.mass[pr.j] / ((rho[pr.i] + rho[pr.j]) * 0.5)),
                (self.fb, float(F(cb)), lambda pr: np.asarray(bvel, F).astype(np.float64)[pr.j],
                 lambda pr: np.asarray(bvol, F).astype(np.float64)[pr.j] * self.rho0[pr.i] / rho[pr.i])):
            if coef == 0:
                continue
            dv = v[pr.i] - vj(pr)
            vr = (pr.x * dv).sum(1)
            vrA = (np.abs(pr.x) * np.abs(dv)).sum(1)
            amb[pr.i[(np.abs(vr) <= 8 * U * vrA) & (vrA > 0)]] = True   # vrA = 0 (self, equal velocities): exactly 0 both ways
            on = (vr < 0) | (not vr_gate)
            mu = h * vr / (pr.d2 + eta2)
            muA = h * vrA / (pr.d2 + eta2)
            m = scale(pr)
            w = np.where(on, coef * (c_s * al * mu - be * mu * mu) * m, 0.0)
            wA = np.where(on, abs(coef) * (abs(c_s * al) * muA + abs(be) * muA * muA) * np.abs(m), 0.0)
            a, aA, aK = self._grad_terms(pr, w, wA)
            val += _sum(N, pr.i, a)
            A += _sum(N, pr.i, aA)
            K += _sum(N, pr.i, aK)
            n += self._n(pr)
        return Ref(val, A, K, n), amb

    def xsph(self, vel, dens, cf, cb, inv_dt, bvel, bvol):
        """XSPHViscosity (xsph_viscosity.rs:30-95): inv_dt [sum_j cf W_ij m_j / rho_j (v_j - v_i) (same fluid)
        + sum_b cb W_ib vol_b rho0_i / rho_i (v_b - v_i)]."""
        N = self.N
        v = np.asarray(vel, F).astype(np.float64)
        rho = np.asarray(dens, F).astype(np.float64)
        s = float(F(inv_dt))
        sf = self.ff.subset(self.fid[self.ff.i] == self.fid[self.ff.j])
        w, _, we = self._w(sf)
        c = float(F(cf)) * self.mass[sf.j] / rho[sf.j]
        dv = v[sf.j] - v[sf.i]
        val = _sum(N, sf.i, (c * w)[:, None] * dv)
        A = _sum(N, sf.i, np.abs(c * w)[:, None] * np.abs(dv))
        K = _sum(N, sf.i, (np.abs(c) * we)[:, None] * np.abs(dv))
        n = self._n(sf).astype(np.float64)
        if cb != 0:
            fb = self.fb
            wb, _, wbe = self._w(fb)
            mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * self.rho0[fb.i]
            cbv = float(F(cb)) * mb / rho[fb.i]
            dvb = np.asarray(bvel, F).astype(np.float64)[fb.j] - v[fb.i]
            val += _sum(N, fb.i, (cbv * wb)[:, None] * dvb)
            A += _sum(N, fb.i, np.abs(cbv * wb)[:, None] * np.abs(dvb))
            K += _sum(N, fb.i, (np.abs(cbv) * wbe)[:, None] * np.abs(dvb))
            n += self._n(fb)
        return Ref(val * s, A * s, K * s, n)


def _cohesion(r, h):
    """Akinci's cohesion spline C(r) (akinci2013_surface_tension.rs:71-88): value, absolute evaluation, kernel error."""
    norm = 32.0 / (np.pi * h ** 9)

    def f(r):
        hr = (h - r) ** 3 * r ** 3
        return norm * np.where(r <= h / 2, 2 * hr - h ** 6 / 64, np.where(r <= h, hr, 0.0))
    fa = norm * np.where(r <= h, 2 * (h + r) ** 3 * r ** 3 + h ** 6 / 64, 0.0)
    v = f(r)
    e = np.maximum(np.abs(f(r * (1 + C_K * U)) - v), np.abs(f(r * (1 - C_K * U)) - v)) + C_K * U * fa
    return v, fa, e


def _adhesion(r, h):
    """Akinci's adhesion kernel (akinci2013_surface_tension.rs:90-111): 0.007 / h^3.25 (-4 r^2 / h + 6 r - 2 h)^(1/4) on
    (h/2, h].  Its error bound perturbs the radicand by its own absolute evaluation too: the fourth root is not Lipschitz
    at the ends of its support."""
    norm = 0.007 / h ** 3.25
    on = (r > h / 2) & (r <= h)
    x = -4 * r * r / h + 6 * r - 2 * h
    xa = 4 * r * r / h + 6 * r + 2 * h
    root = lambda y: norm * np.maximum(y, 0.0) ** 0.25  # noqa: E731
    v = np.where(on, root(x), 0.0)

    def at(rr):
        onr = (rr > h / 2) & (rr <= h)
        return np.where(onr, root(-4 * rr * rr / h + 6 * rr - 2 * h), 0.0)
    e = np.maximum(np.abs(at(r * (1 + C_K * U)) - v), np.abs(at(r * (1 - C_K * U)) - v))
    e += np.where(on, np.maximum(np.abs(root(x + C_K * U * xa) - v), np.abs(root(x - C_K * U * xa) - v)), 0.0)
    return v, np.where(on, norm * xa ** 0.25, 0.0), e
