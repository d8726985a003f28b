"""Float64 restatement of single DFSPH and IISPH gather passes and of the WCSPH, He2014, DFSPHViscosity and Becker2009
plugins' passes, each with the scale its float32 evaluation's error is measured against.

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

Cites (reference src/): kernel/*.rs, solver/pressure/dfsph_solver.rs, solver/pressure/iisph_solver.rs, solver/viscosity/xsph_viscosity.rs,
solver/surface_tension/{akinci2013,he2014,wcsph}_surface_tension.rs, solver/elasticity/becker2009_elasticity.rs, as restated in SURVEY.md Appendix A.
"""
import itertools
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
    # IISPH (iisph_solver.rs).  A pass whose term carries the gradient twice (g^2 |x|^2) counts its normalisation and its
    # 6.2 + dx twice.
    # dii: factor -dt dt / (rho rho) 3, m_j factor 1 (boundary vol_b rho0 factor 2), g x 1, fma with x 1 + dx 1, g 6.2, margin 1
    iisph_dii=C_NORM + 14,
    # aii: g and dx twice 14.4, factor dt dt m_i / (rho rho) 4, g dx 1, dii - g dx factor 2, * g dx 1, dot sums 2,
    # fma with m_j (boundary vol_b rho0: 1 more) 2, margin 3.6
    iisph_aii=2 * C_NORM + 30,
    # dij_pjl: prho = p / (rho rho) 2, -m_j prho_j 1, g x 1, fma with x 1 + dx 1, g 6.2, dt dt 1, * dt^2 1, margin 1.8
    iisph_dij_pjl=C_NORM + 16,
    # next pressure: the sum's term as aii's 14.4 + 2 + 2 + 1 + 2, dji_f = dt dt m_i / (rho rho) p_i 5, dij_i - s_j 1, s_j's
    # own fma 1 (carried in A through |dii_j p_j| + |dij_pjl_j|); then rho0 - pred 1, - sum 1, / aii 1, omega * 1,
    # (1 - omega) * p 2, + 1; margin 3.6
    iisph_pressure=2 * C_NORM + 38,
    # velocity: prho 2, prho_i + prho_j 1, dt m_j 1, * 1, g x 1, fma with x 1 + dx 1, g 6.2, vc - sum 1, v + vc 1, boundary
    # c dt 1; margin 1.8
    iisph_velocity=C_NORM + 18,
    # Surface tension plugins (surface_tension/*.rs), over same-fluid contacts.
    # WCSPH: c = -cf W m_j / m_i: -cf W 1, * m_j 1, / m_i 1; fma with x 1 + dx 1; margin 3
    wcsph=C_NORM + 8,
    # He2014 colours: W m_j 1, / rho_j 1 (boundary: W vol_b 1); margin 2
    he2014_color=C_NORM + 4,
    # He2014 gradc, per component before the square: c = g c_j m_j / rho_j 3, g 6.2, fma with x 1 + dx 1; margin 1.8.  The
    # division by c_i and the square are carried explicitly (Passes.he2014_gradc)
    he2014_gradc=C_NORM + 13,
    # He2014 force: fluid m_i / rho_i 1, * m_j 1, / rho_j 1, g_i + g_j 1, * 1, g * 1, g 6.2, * x 1 + dx 1, * k 1, k = cf / (2 m_i)
    # 1; boundary vol_b rho0 1, / rho0 1, * g_i 1, * cb 1, s * x 1, / m_i 1, acc + 1; margin 2.8
    he2014_force=C_NORM + 18,
    # DFSPHViscosity.  G = grad W m_j / (2 rho_i): g 6.2, * x 1 + dx 1, s = m_j / (2 rho_i) 1, * s 1, margin 1.8; the
    # matrix entries (products of two G, / rho, sums) are bounded from it in Passes.visc_matrix
    visc_matrix=C_NORM + 12,
    # strain rate: G as above 11 + vv = fma(a, dt, v) 1, vv_j - vv_i 1, products and the pair sum 2, margin 2
    visc_rate=C_NORM + 16,
    # acceleration: g 6.2 + dx 1, u_i + u_j 1, * m_j / 2 1, gradient^T products and sums 3, * m_i inv_dt 2, acc + 1,
    # margin 2.8 (u's own error is carried in K)
    visc_accel=C_NORM + 18,
    # Becker2009 elasticity (becker2009_elasticity.rs), over the rest contacts, always with the cubic spline.
    # rest volume, checked as m_i / vol0 against the sum: 2 m_j W 1 (2 exact), m_i / sum 1, its inverse read back 1; margin 2
    el_volume=C_NORM + 5,
    # A_pq entry: p = x_j - x_i 1, q = x0_j - x0_i 1, coeff = W m_j 1, q coeff 1, p q 1; margin 2
    el_apq=C_NORM + 7,
    # grad_tr entry: a = g vol0_j x0 (g 6.2, * vol0 1, * x0 1 + dx 1), u = R^T p - q (p 1, three products and two sums 3,
    # q 1, - 1: carried in A through |R|^T |p| + |q|), a u 1; margin 2.8
    el_grad_tr=C_NORM + 18,
    # force term: grad 6.2 + dx 1, * vol0 1, S d (products and sums) 3, G (S d) 3 + 1, * vol0 1, R f 3, R_j f_ij - R_i f_ji 1,
    # * 0.5 / m_i 1; margin 2.8
    el_force=C_NORM + 24,
)
# stress from grad_tr read back, no sum: J = G + I 1, J J^T 3, - 1 1, d0 ex + d1 ey + d1 ez 3, * k 1, * d2 1; margin 2
C_EL_STRESS = 12
# orthonormality of the float32 rotation: each of at most 20 iterations multiplies by an axis-angle rotation built from
# sin / cos and products (<= 8u per entry) in a 3-term product (3u)
C_EL_ORTHO = 20 * 11 + 20
IISPH_AII_GATE = 1.0e-9  # iisph_solver.rs:303: no pressure where |aii| <= 1e-9
# the loop errors: the term's division by rho0 (1), the mean's division by n (1), margin 2; the sum's depth is n
C_ERR = 4
# integration: vc = acc dt (1), margin 1; positions: v + vc, * dt, + P (3), margin 1
C_INTEGRATE = 2
C_POSITIONS = 4


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


def contacts_rows(P, Q, h, allowed, rows, tree=None):
    """The contacts of the points P[rows] only, otherwise as `contacts`: candidates within h (1 + 1e-5) from a k-d tree over
    all of Q (query_ball_point keeps zero distances, so self contacts and coincident points are in), the same float32 test
    and group mask, and the same (i, j) order, so each row's list is term for term the one `contacts` gives it.  i and j
    stay global indices.  tree: a cKDTree over Q to reuse."""
    h32 = F(h)
    h2 = F(h32 * h32)
    rows = np.asarray(rows, np.int64)
    if len(Q) == 0 or len(rows) == 0:
        z = np.zeros(0, np.int64)
        return Pairs(z, z, np.zeros((0, 3)))
    tq = cKDTree(Q.astype(np.float64)) if tree is None else tree
    hits = tq.query_ball_point(P[rows].astype(np.float64), float(h32) * (1.0 + 1e-5), workers=-1)
    ln = np.fromiter(map(len, hits), np.int64, len(hits))
    i = np.repeat(rows, ln)
    j = np.fromiter(itertools.chain.from_iterable(hits), np.int64, int(ln.sum()))
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
    BP / bid: boundary positions and boundary of each, allowed_ff / allowed_fb: interaction-group masks over (i, j).

    rows: build the fluid-fluid and fluid-boundary contacts of these particles only (contacts_rows).  Every pass then runs
    unchanged over global indices and is exact, term for term, at the rows; elsewhere its sums are partial and meaningless.
    Boundary-boundary contacts stay complete.  brows: the boundary particles all of whose fluid contacts belong to rows, so
    that sums onto boundary particles are whole there."""

    def __init__(self, h, P, fid, rho0, mass, BP, bid, allowed_ff=None, allowed_fb=None, allowed_bb=None, kw=0, kg=0, rows=None):
        self.h = float(F(h))
        self.P, self.fid = P, fid
        self.rho0 = np.asarray(rho0, F).astype(np.float64)
        self.mass = np.asarray(mass, F).astype(np.float64)
        self.BP, self.bid = BP, bid
        self.kw, self.kg = kw, kg
        self.grad_t = grad_threshold(kg, self.h)   # the gradient's zero threshold on d^2
        self.N = len(P)
        every = lambda i, j: np.ones(len(i), bool)  # noqa: E731
        self.allowed_ff = allowed_ff or every
        self._halo = None
        if rows is None:
            self.rows = self.brows = None
            self.ff = contacts(P, P, self.h, self.allowed_ff, same=True)
            self.fb = contacts(P, BP, self.h, allowed_fb or every)
        else:
            self.rows = np.unique(np.asarray(rows, np.int64))
            self._tree = cKDTree(P.astype(np.float64))
            self.ff = contacts_rows(P, P, self.h, self.allowed_ff, self.rows, tree=self._tree)
            self.fb = contacts_rows(P, BP, self.h, allowed_fb or every, self.rows)
            # a boundary particle is whole when no fluid particle outside rows lies within reach of it
            inside = np.zeros(self.N, bool)
            inside[self.rows] = True
            near = self._tree.query_ball_point(np.asarray(BP, np.float64), self.h * (1.0 + 1e-5), workers=-1) if len(BP) else []
            self.brows = np.array([k for k, hit in enumerate(near) if inside[hit].all()], np.int64)
        self.bb = contacts(BP, BP, self.h, allowed_bb or every, same=True)
        self.nf = np.bincount(self.ff.i, minlength=self.N)
        self.nb = np.bincount(self.fb.i, minlength=self.N)

    def halo(self):
        """Rows mode: the fluid-fluid contacts of the rows and of all their neighbours (for a pass that reads a gathered
        quantity of its neighbours, such as Akinci's normals).  Full mode: ff."""
        if self.rows is None:
            return self.ff
        if self._halo is None:
            self._halo = contacts_rows(self.P, self.P, self.h, self.allowed_ff, np.unique(self.ff.j), tree=self._tree)
        return self._halo

    # ambiguous float decisions: the gradient's zero threshold
    def ambiguous(self, pairs=None):
        """Particles with a contact whose squared distance lies within the float32 d2's rounding of the gradient's zero
        threshold: there the kernel may take either side."""
        t = self.grad_t
        out = np.zeros(self.N, bool)
        for pr in ([self.ff, self.fb] if pairs is None else pairs):
            near = np.abs(pr.d2 - t) <= 8 * U * t
            out[pr.i[near]] = True
        return out

    def _g(self, pr):
        g, ga, ge = kernel(self.kg, "g", pr.r, self.h)
        z = pr.d2 <= self.grad_t
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

    def akinci(self, dens, gamma, adhesion, bvol, rho_i_for_j=False, ff=None, fb=None):
        """Akinci2013SurfaceTension (akinci2013_surface_tension.rs:43-192): normals n_i = h sum_j (m_j / rho_j) grad W_ij over
        the same fluid, then the fluid force sum_j kij (-gamma (n_i - n_j) - gamma m_j C(r) x_ij / r), kij = 2 rho0 /
        (rho_i + rho_j), and the adhesion -adh vol_b rho0 A(r) x_ib / r.  rho_i_for_j: the normals divide by rho_i instead
        of rho_j.  The normals' own error bound is carried into the force's bound.  In rows mode the normals come from the
        halo's contacts (the neighbours' normals are sums over their own lists)."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        N, h = self.N, self.h
        same = self.fid[ff.i] == self.fid[ff.j]
        sf = ff.subset(same)
        rho = np.asarray(dens, F).astype(np.float64)
        nf_ = sf if self.rows is None else self.halo()
        nf_ = nf_.subset(self.fid[nf_.i] == self.fid[nf_.j])
        a, aA, aK = self._grad_terms(nf_, self.mass[nf_.j] / rho[nf_.i if rho_i_for_j else nf_.j])
        nrm = h * _sum(N, nf_.i, a)
        nn = self._n(sf).astype(np.float64)
        e_n = h * ((self._n(nf_) + C_PASS["normals"])[:, None] * U * _sum(N, nf_.i, aA) + _sum(N, nf_.i, aK))
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
        return self.update_boundary_force(kappa, bvol, inv_dt, pressure=True, scale_m_inv_dt=scale_m_inv_dt)

    def update_boundary_force(self, kappa, bvol, inv_dt, pressure=True, scale_m_inv_dt=True):
        """The force an update puts on boundary particles, per boundary particle.  Pressure update (dfsph_solver.rs:267-272):
        (k_i vol_b rho0_i inv_dt g_ib) inv_dt m_i x_ib over contacts with k_i > 0.  Divergence update (:400-406):
        (k_i vol_b rho0_i g_ib) inv_dt m_i x_ib, where inv_dt is the previous step's (0 on the first step) and k_i =
        div_i alpha_i >= 0.  scale_m_inv_dt = False drops the outer inv_dt m_i."""
        fb = self.fb
        k = np.asarray(kappa, F).astype(np.float64)[fb.i]
        s = float(F(inv_dt))
        mb = np.asarray(bvol, F).astype(np.float64)[fb.j] * self.rho0[fb.i]
        inner = np.where(k > 0, k * mb * s, 0.0) if pressure else k * mb
        w = inner * ((s * self.mass[fb.i]) if scale_m_inv_dt else 1.0)
        return self._on_boundary(fb, *self._grad_terms(fb, w))

    def loop_error(self, kind, x, c_pass=0, mutant=None, block=128):
        """The error a DFSPH Jacobi loop breaks on (dfsph_solver.rs:153-158, 347-352): per particle e_i = max(div_i, 0) / rho0
        (kind "divergence"; 0 under the 20-contact gate, still counted) or pred_i < rho0 ? 0 : pred_i / rho0 - 1 (kind
        "density"); per fluid the mean over its particles; over fluids the maximum, empty fluids skipped, and 0.  Returns
        (value, bound).
        x: the float32 values read back (the reduction fed its own inputs), or a Ref of the pass (end to end: the pass
        bound, at c_pass, is carried through the sum; both terms are 1 / rho0-Lipschitz in their input and continuous at
        their gates, so no particle needs excluding).
        The float32 reduction: each term rounds once or twice (x / rho0, then - 1, which cancels: its rounding is relative
        to q = x / rho0), the sum of n terms in any order (n - 1) u sum |e|, and the division by n.
        mutant: error_mean_over_all_fluids, error_drops_last_block (of `block` particles), error_unclamped (density)."""
        end = isinstance(x, Ref)
        v = x.value if end else _f64(x)
        b = (x.bound(c_pass) if end else np.zeros(self.N)) / self.rho0
        if kind == "divergence":
            e = np.maximum(v, 0.0) / self.rho0
            a = e
        else:
            q = v / self.rho0
            on = (v >= self.rho0) | (mutant == "error_unclamped")
            e = np.where(on, q - 1.0, 0.0)
            a = np.where(on, np.abs(q) + np.abs(e), 0.0)
        keep = np.ones(self.N, bool)
        if mutant == "error_drops_last_block" and self.N:
            keep[(self.N - 1) // block * block:] = False
        groups = [np.arange(self.N)] if mutant == "error_mean_over_all_fluids" else \
            [np.nonzero(self.fid == f)[0] for f in np.unique(self.fid)]
        val, bound = 0.0, 0.0
        for sel in groups:
            n = len(sel)
            val = max(val, e[sel[keep[sel]]].sum() / n)
            # the maximum over fluids is 1-Lipschitz in each: the bound of the maximum is the largest bound
            bound = max(bound, ((n + C_ERR) * U * np.abs(e[sel]).sum() + U * a[sel].sum() + b[sel].sum()) / n)
        return val, bound

    def loop_error_structural(self, kind, x, block, second, mutant=None):
        """loop_error fed the float32 values read back, over all particles, against the bound of the reduction tree the
        engine runs (structural_depth) instead of the any-order (n + 4) u sum |e|: (D + C_ERR) u sum |e| + u sum a, per
        fluid over n.  block: threads per block of the pass (PASS_T, or NBR_T for the neighbour search's fused first
        evaluation); second: threads of the block that sums the partials (PASS_T for a pass's last block, 256 for
        k_reduce_partials).  mutant: error_drops_blocks_past_65535 (every partial of block >= 65536 lost).  Returns
        (value, bound, D)."""
        v = _f64(x)
        if kind == "divergence":
            e = np.maximum(v, 0.0) / self.rho0
            a = e
        else:
            q = v / self.rho0
            on = v >= self.rho0
            e = np.where(on, q - 1.0, 0.0)
            a = np.where(on, np.abs(q) + np.abs(e), 0.0)
        keep = np.ones(self.N, bool)
        if mutant == "error_drops_blocks_past_65535":
            keep[65536 * block:] = False
        D = structural_depth(self.N, block, second)
        g = D * U / (1.0 - D * U)
        val, bound = 0.0, 0.0
        for f in np.unique(self.fid):
            sel = np.nonzero(self.fid == f)[0]
            n = len(sel)
            val = max(val, e[sel[keep[sel]]].sum() / n)
            bound = max(bound, ((g + C_ERR * U) * np.abs(e[sel]).sum() + U * a[sel].sum()) / n)
        return val, bound, D

    def integrate(self, acc, dt):
        """The velocity change of the integration (dfsph_solver.rs:505-518): vc = acc dt, one float32 rounding."""
        a = _f64(acc) * float(F(dt))
        return Ref(a, np.abs(a), np.zeros_like(a), np.zeros(self.N))

    def positions(self, P, V, vc, dt):
        """update_positions (dfsph_solver.rs:411-420): P' = P + (v + vc) dt, fed the float32 P, v and vc; three float32
        roundings (v + vc, * dt, + P), each relative to its operands."""
        P, s, dt = _f64(P), _f64(V) + _f64(vc), float(F(dt))
        return Ref(P + s * dt, np.abs(P) + (np.abs(_f64(V)) + np.abs(_f64(vc))) * abs(dt), np.zeros_like(P), np.zeros(self.N))

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

    # ---- IISPH (iisph_solver.rs) ----------------------------------------------------------------------------------------
    # Every input is the float32 array the kernel reads (densities, pressures, dii, aii, dij_pjl read back), so the kernels'
    # pre-combined quantities (prho = p / rho^2, s_j = dii_j p_j + dij_pjl_j, dji_f = dt^2 m_i / rho_i^2 p_i) are restated
    # from their parts here and their roundings are counted in C_PASS.
    def _pseudo_mass(self, fb, bvol, rho0_b):
        return _f64(bvol)[fb.j] * (self.rho0 if rho0_b is None else rho0_b)[fb.i]

    def iisph_dii(self, dens, bvol, dt, rho0_b=None, ff=None, fb=None):
        """dii_i = -dt^2 / rho_i^2 [sum_j m_j grad W_ij + sum_b vol_b rho0_i grad W_ib] (iisph_solver.rs:144-186)."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho, dt = _f64(dens), float(F(dt))
        fac = -dt * dt / (rho * rho)
        a, aA, aK = self._grad_terms(ff, self.mass[ff.j] * fac[ff.i])
        b, bA, bK = self._grad_terms(fb, self._pseudo_mass(fb, bvol, rho0_b) * fac[fb.i])
        N = self.N
        return Ref(_sum(N, ff.i, a) + _sum(N, fb.i, b), _sum(N, ff.i, aA) + _sum(N, fb.i, bA),
                   _sum(N, ff.i, aK) + _sum(N, fb.i, bK), (self._n(ff) + self._n(fb)).astype(np.float64))

    def _quadratic(self, pr, w, u, uA, cf):
        """Per contact w [g (u . x) + cf g^2 |x|^2] (aii's and the pressure sum's term; cf: d_ji's factor), its absolute
        evaluation and its kernel part (g enters twice)."""
        g, _, ge = self._g(pr)
        ux, uxA = (u * pr.x).sum(1), (uA * np.abs(pr.x)).sum(1)
        wa, ca = np.abs(w), np.abs(cf)
        t = w * (g * ux + cf * g * g * pr.d2)
        tA = wa * (np.abs(g) * uxA + ca * g * g * pr.d2)
        tK = wa * (uxA + ca * (2 * np.abs(g) + ge) * pr.d2) * ge
        return t, tA, tK

    def iisph_aii(self, dens, dii, bvol, dt, rho0_b=None, dji_mass=None, ff=None, fb=None):
        """aii = sum_j m_j (dii_i - d_ji) . grad W_ij + sum_b vol_b rho0_i (dii_i - d_ji) . grad W_ib with d_ji = dt^2 m_i /
        rho_i^2 grad W_ij (iisph_solver.rs:188-233).  dii: the float32 dii the kernel read.  dji_mass: per fluid contact, the
        mass d_ji uses (default m_i)."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho, d, dt = _f64(dens), _f64(dii), float(F(dt))
        fac = dt * dt / (rho * rho)
        mi = self.mass[ff.i] if dji_mass is None else dji_mass
        N = self.N
        val, A, K = np.zeros(N), np.zeros(N), np.zeros(N)
        for pr, w, cf in ((ff, self.mass[ff.j], -fac[ff.i] * mi),
                          (fb, self._pseudo_mass(fb, bvol, rho0_b), -fac[fb.i] * self.mass[fb.i])):
            t, tA, tK = self._quadratic(pr, w, d[pr.i], np.abs(d[pr.i]), cf)
            val += _sum(N, pr.i, t)
            A += _sum(N, pr.i, tA)
            K += _sum(N, pr.i, tK)
        return Ref(val, A, K, (self._n(ff) + self._n(fb)).astype(np.float64))

    def iisph_dij_pjl(self, dens, press, dt, prho_i=False, ff=None):
        """dij_pjl_i = dt^2 sum_j -m_j p_j / rho_j^2 grad W_ij over fluid contacts (iisph_solver.rs:235-268).  press: the
        pressures of the previous iteration.  prho_i: p_i / rho_i^2 in place of p_j / rho_j^2."""
        ff = self.ff if ff is None else ff
        rho, p, dt = _f64(dens), _f64(press), float(F(dt))
        prho = p / (rho * rho)
        a, aA, aK = self._grad_terms(ff, -dt * dt * self.mass[ff.j] * prho[ff.i if prho_i else ff.j])
        N = self.N
        return Ref(_sum(N, ff.i, a), _sum(N, ff.i, aA), _sum(N, ff.i, aK), self._n(ff).astype(np.float64))

    def _pressure_sum(self, dens, press, dii, dij, bvol, dt, rho0_b=None, dji_mass=None, s_dii_p=True, boundary=True,
                      ff=None, fb=None):
        """sum_i = sum_j m_j (dij_pjl_i - s_j + d_ji p_i) . grad W_ij + sum_b vol_b rho0_i dij_pjl_i . grad W_ib, with
        s_j = dii_j p_j + dij_pjl_j (iisph_solver.rs:296-322): (value, A, K, n)."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho, p, d, dj, dt = _f64(dens), _f64(press), _f64(dii), _f64(dij), float(F(dt))
        s = dj + (d * p[:, None] if s_dii_p else 0.0)
        sA = np.abs(dj) + (np.abs(d) * np.abs(p)[:, None] if s_dii_p else 0.0)
        mi = self.mass[ff.i] if dji_mass is None else dji_mass
        cf = dt * dt * mi / (rho[ff.i] * rho[ff.i]) * p[ff.i]
        N = self.N
        t, tA, tK = self._quadratic(ff, self.mass[ff.j], dj[ff.i] - s[ff.j], np.abs(dj[ff.i]) + sA[ff.j], cf)
        val, A, K = _sum(N, ff.i, t), _sum(N, ff.i, tA), _sum(N, ff.i, tK)
        if boundary:
            b, bA, bK = self._grad_terms(fb, self._pseudo_mass(fb, bvol, rho0_b))
            val += (_sum(N, fb.i, b) * dj).sum(1)
            A += (_sum(N, fb.i, bA) * np.abs(dj)).sum(1)
            K += (_sum(N, fb.i, bK) * np.abs(dj)).sum(1)
        return val, A, K, (self._n(ff) + self._n(fb)).astype(np.float64)

    def iisph_next_pressure(self, dens, pred, press, aii, dii, dij, bvol, dt, omega, pred_err=None, relax=True, **kw):
        """p_i' = (1 - omega) p_i + omega (rho0_i - pred_i - sum_i) / aii_i, 0 where |aii_i| <= 1e-9 or p_i' <= 0
        (iisph_solver.rs:270-353).  Returns (Ref, unclamped): the clamp is a float decision, so the caller excludes particles
        whose unclamped value lies within its bound of 0.  pred_err: an absolute error of pred (when pred is itself a
        reference value rather than the float32 array the kernel read).  relax = False drops (1 - omega) p_i.
        The error of (rho0 - pred) - sum is carried through A rather than taken relative to the result: the two cancel."""
        S, SA, SK, n = self._pressure_sum(dens, press, dii, dij, bvol, dt, **kw)
        p, a, pr = _f64(press), _f64(aii), np.asarray(pred, np.float64)
        om = float(F(omega))
        on = np.abs(a) > IISPH_AII_GATE   # an exact decision on the float32 input
        sa = np.where(on, np.abs(a), 1.0)
        raw = (1.0 - om) * p * relax + om * (self.rho0 - pr - S) / np.where(on, a, 1.0)
        A = (1.0 - om) * np.abs(p) * relax + om * (self.rho0 + np.abs(pr) + SA) / sa
        K = om * (SK + (0.0 if pred_err is None else pred_err)) / sa
        val = np.where(on, np.maximum(raw, 0.0), 0.0)
        return Ref(val, np.where(on, A, 0.0), np.where(on, K, 0.0), n), np.where(on, raw, np.nan)

    def iisph_density_error(self, dens, pred, press, aii, dii, dij, bvol, dt, omega, c_pass, count_clamped=False, relax=True,
                            **kw):
        """The pressure iteration's density error: per fluid, the sum over its particles with p_i' > 0 of
        (-sum_i - aii_i p_i') / rho0, divided by the fluid's particle count, then the maximum over fluids and 0 (the
        kernel's block partials and read_error).  Returns (value, bound, ambiguous): the bound carries the errors of sum_i and
        p_i', and for particles whose p_i' lies within its bound of 0 (either side of the clamp) the whole term.
        count_clamped: clamped particles add -sum_i / rho0 too."""
        S, SA, SK, n = self._pressure_sum(dens, press, dii, dij, bvol, dt, **kw)
        ref, raw = self.iisph_next_pressure(dens, pred, press, aii, dii, dij, bvol, dt, omega, relax=relax, **kw)
        a = _f64(aii)
        on = np.abs(a) > IISPH_AII_GATE
        bp = ref.bound(c_pass)
        amb = on & (np.abs(np.nan_to_num(raw)) <= bp)
        pos = on & (np.nan_to_num(raw) > 0)
        e = (-S - a * ref.value) / self.rho0
        eS = (n + c_pass) * U * SA + SK
        ee = (eS + np.abs(a) * bp + 3 * U * (np.abs(S) + np.abs(a * ref.value))) / self.rho0
        take = pos | (count_clamped & on)
        val, bound = 0.0, 0.0
        for f in np.unique(self.fid):
            sel = self.fid == f
            nf = sel.sum()
            ef = np.where(take & sel & ~amb, e, 0.0)
            slack = np.where(sel & take & ~amb, ee, 0.0) + np.where(sel & amb, np.abs(e) + ee, 0.0)
            v = ef.sum() / nf
            b = (slack.sum() + (nf + 2) * U * np.abs(np.where(sel & (take | amb), e, 0.0)).sum()) / nf
            # max over fluids is 1-Lipschitz in each: the bound of the maximum is the largest bound
            val, bound = max(val, v), max(bound, b)
        return val, bound, int(amb.sum())

    def iisph_velocity(self, dens, press, v0, bvol, dt, rho0_b=None, prho_i_twice=False, ff=None, fb=None):
        """v0 - dt sum_j m_j (p_i / rho_i^2 + p_j / rho_j^2) grad W_ij - dt sum_b vol_b rho0_i p_i / rho_i^2 grad W_ib
        (iisph_solver.rs:355-420: the velocity change added to the velocity).  prho_i_twice: p_i / rho_i^2 for both."""
        ff = self.ff if ff is None else ff
        fb = self.fb if fb is None else fb
        rho, p, dt = _f64(dens), _f64(press), float(F(dt))
        prho = p / (rho * rho)
        pj = prho[ff.i] if prho_i_twice else prho[ff.j]
        a, aA, aK = self._grad_terms(ff, dt * self.mass[ff.j] * (prho[ff.i] + pj),
                                     dt * self.mass[ff.j] * (np.abs(prho[ff.i]) + np.abs(pj)))
        b, bA, bK = self._grad_terms(fb, dt * self._pseudo_mass(fb, bvol, rho0_b) * prho[fb.i])
        v0 = _f64(v0)
        N = self.N
        return Ref(v0 - _sum(N, ff.i, a) - _sum(N, fb.i, b), np.abs(v0) + _sum(N, ff.i, aA) + _sum(N, fb.i, bA),
                   _sum(N, ff.i, aK) + _sum(N, fb.i, bK), (self._n(ff) + self._n(fb) + 1).astype(np.float64))

    def iisph_boundary_force(self, dens, press, bvol, rho0_b=None, with_mass=True):
        """The force the pressure puts on boundary particles (iisph_solver.rs:399-401): per boundary particle,
        sum_i m_i vol_b rho0_i p_i / rho_i^2 grad W_ib.  with_mass = False drops m_i."""
        fb = self.fb
        rho, p = _f64(dens), _f64(press)
        w = self._pseudo_mass(fb, bvol, rho0_b) * (p / (rho * rho))[fb.i] * (self.mass[fb.i] if with_mass else 1.0)
        return self._on_boundary(fb, *self._grad_terms(fb, w))

    # ---- surface tension plugins (surface_tension/*.rs) -----------------------------------------------------------------
    # Fluid sums run over contacts of the particle's own fluid (self included: x_ii = 0); every input is the float32 array
    # the kernel read (densities, and the colours and gradc read back).
    def _same(self):
        return self.ff.subset(self.fid[self.ff.i] == self.fid[self.ff.j])

    def _vec_sum(self, pr, t, tA, tK, n=None):
        N = self.N
        return Ref(_sum(N, pr.i, t), _sum(N, pr.i, tA), _sum(N, pr.i, tK), self._n(pr).astype(np.float64) if n is None else n)

    def wcsph(self, cf, inverted_mass_ratio=False):
        """WCSPHSurfaceTension's fluid term (wcsph_surface_tension.rs:45-63): sum_j -cf W_ij m_j / m_i x_ij.
        inverted_mass_ratio: m_i / m_j."""
        sf = self._same()
        w, _, we = self._w(sf)
        ratio = self.mass[sf.i] / self.mass[sf.j] if inverted_mass_ratio else self.mass[sf.j] / self.mass[sf.i]
        c = -float(F(cf)) * ratio
        return self._vec_sum(sf, (c * w)[:, None] * sf.x, np.abs(c * w)[:, None] * np.abs(sf.x), (np.abs(c) * we)[:, None] * np.abs(sf.x))

    def he2014_colors(self, dens, bvol, boundary=True):
        """He2014's colours (he2014_surface_tension.rs:40-75): sum_j W_ij m_j / rho_j + sum_b W_ib vol_b."""
        sf, fb, N = self._same(), self.fb, self.N
        w, _, we = self._w(sf)
        c = self.mass[sf.j] / _f64(dens)[sf.j]
        val, A, K = _sum(N, sf.i, c * w), _sum(N, sf.i, np.abs(c * w)), _sum(N, sf.i, c * we)
        n = self._n(sf)
        if boundary:
            wb, _, wbe = self._w(fb)
            vb = _f64(bvol)[fb.j]
            val, A, K = val + _sum(N, fb.i, vb * wb), A + _sum(N, fb.i, np.abs(vb * wb)), K + _sum(N, fb.i, vb * wbe)
            n = n + self._n(fb)
        return Ref(val, A, K, n.astype(np.float64))

    def he2014_gradc(self, dens, colors, c_pass, divide_by_cj=False):
        """He2014's squared colour-gradient norm (he2014_surface_tension.rs:77-105): |sum_j grad W_ij c_j m_j / rho_j / c_i|^2.
        The vector sum cancels in the interior, so its error is bounded per component and carried through the division
        and the square explicitly (as in den); the Ref's A is 0 and K the whole bound.  divide_by_cj: each term divided by
        its own c_j instead of the sum by c_i."""
        sf, N = self._same(), self.N
        c = _f64(colors)
        wt = self.mass[sf.j] / _f64(dens)[sf.j] * (1.0 if divide_by_cj else c[sf.j])
        a, aA, aK = self._grad_terms(sf, wt)
        n = self._n(sf).astype(np.float64)
        gs = _sum(N, sf.i, a)
        e_gs = (n + c_pass)[:, None] * U * _sum(N, sf.i, aA) + _sum(N, sf.i, aK)
        ci = np.ones(N) if divide_by_cj else np.abs(c)
        q = gs / ci[:, None]
        e_q = e_gs / ci[:, None] + U * np.abs(q)
        val = (q * q).sum(1)
        e = (2 * np.abs(q) * e_q + e_q * e_q).sum(1) + 4 * U * val
        return Ref(val, np.zeros(N), e, n)

    def _he2014_boundary_terms(self, dens, gradc, cb, bvol):
        """Per fluid-boundary contact f = cb / 4 grad W_ib m_i / rho_i vol_b g_i (the boundary loop of he2014_surface_tension.rs:131-178)."""
        fb = self.fb
        w = float(F(cb)) * 0.25 * self.mass[fb.i] / _f64(dens)[fb.i] * _f64(bvol)[fb.j] * _f64(gradc)[fb.i]
        return fb, self._grad_terms(fb, w)

    def he2014_force(self, dens, gradc, cf, cb, bvol, gradc_i_twice=False):
        """He2014's acceleration (he2014_surface_tension.rs:131-178): cf / (2 m_i) sum_j grad W_ij m_i / rho_i m_j / rho_j
        (g_i + g_j) / 2 over the same fluid, plus the boundary term f / m_i.  gradc_i_twice: g_i + g_i."""
        sf, N = self._same(), self.N
        g, rho = _f64(gradc), _f64(dens)
        gj = g[sf.i] if gradc_i_twice else g[sf.j]
        base = float(F(cf)) / (2.0 * self.mass[sf.i]) * self.mass[sf.i] / rho[sf.i] * self.mass[sf.j] / rho[sf.j] * 0.5
        a, aA, aK = self._grad_terms(sf, base * (g[sf.i] + gj), np.abs(base) * (np.abs(g[sf.i]) + np.abs(gj)))
        ref = self._vec_sum(sf, a, aA, aK)
        if cb != 0:
            fb, (b, bA, bK) = self._he2014_boundary_terms(dens, gradc, cb, bvol)
            mi = self.mass[fb.i][:, None]
            ref = Ref(ref.value + _sum(N, fb.i, b / mi), ref.A + _sum(N, fb.i, bA / mi), ref.K + _sum(N, fb.i, bK / mi),
                      ref.n + self._n(fb))
        return ref

    # ---- DFSPHViscosity (viscosity/dfsph_viscosity.rs) -----------------------------------------------------------------
    def _visc_grads(self, dens):
        """Same-fluid contacts and, per contact, G = grad W_ij m_j / (2 rho_i), its absolute evaluation and kernel part."""
        sf = self._same()
        g, _, ge = self._g(sf)
        s = self.mass[sf.j] / (2.0 * _f64(dens)[sf.i])
        return sf, (g * s)[:, None] * sf.x, (np.abs(g) * s)[:, None] * np.abs(sf.x), (ge * s)[:, None] * np.abs(sf.x)

    @staticmethod
    def _mat6(G):
        """compute_gradient_matrix (dfsph_viscosity.rs:59-82): rows (2gx,0,0) (0,2gy,0) (0,0,2gz) (gy,gx,0) (gz,0,gx)
        (0,gz,gy), (..., 6, 3)."""
        x, y, z = G[..., 0], G[..., 1], G[..., 2]
        o = np.zeros_like(x)
        return np.stack([np.stack(r, -1) for r in ((2 * x, o, o), (o, 2 * y, o), (o, o, 2 * z), (y, x, o), (z, o, x),
                                                    (o, z, y))], -2)

    def visc_matrix(self, dens, c_pass, by_column=False):
        """The preconditioned 6x6 matrix whose inverse is beta (dfsph_viscosity.rs:133-201), in float64: D = sum_j M_j M_j^T
        / rho_i + M(sum_j G_j) M(sum_j G_j)^T / rho_i with M_j = M(G_j); then column c < 3 of row r scaled by p_r = 1 / D_rr
        (1 where |D_rr| < 1e-6).  Returns (Dt, dDt, p, dp, ambiguous): the bound of each entry of the kernel's float32
        Dt (D's own error plus the float32 p's), p and its relative error, and the particles whose preconditioner switch
        |D_rr| < 1e-6 lies within D_rr's bound.  by_column: column c scaled by p_c instead."""
        sf, G, GA, GK = self._visc_grads(dens)
        N, rho = self.N, _f64(dens)
        n = self._n(sf).astype(np.float64)
        M, MA, MK = self._mat6(G), self._mat6(GA), self._mat6(GK)
        outer = lambda a, b: np.einsum("nrk,nck->nrc", a, b) / rho[sf.i][:, None, None]  # noqa: E731
        sq = lambda t: np.stack([_sum(N, sf.i, t[:, r, :]) for r in range(6)], axis=1)  # noqa: E731
        D1, D1A = sq(outer(M, M)), sq(outer(MA, MA))
        D1K = sq(outer(MA, MK) + outer(MK, MA))
        gs, gsA, gsK = _sum(N, sf.i, G), _sum(N, sf.i, GA), _sum(N, sf.i, GK)
        e_gs = (n + c_pass)[:, None] * U * gsA + gsK
        Ms, MsA, Me = self._mat6(gs), self._mat6(np.abs(gs)), self._mat6(e_gs)
        op = lambda a, b: np.einsum("nrk,nck->nrc", a, b) / rho[:, None, None]  # noqa: E731
        D = D1 + op(Ms, Ms)
        dD = (n + 2 * c_pass + 4)[:, None, None] * U * D1A + D1K + op(MsA, Me) + op(Me, MsA) + op(Me, Me) + \
            8 * U * op(MsA, MsA) + 2 * U * np.abs(D)
        dg = np.diagonal(D, axis1=1, axis2=2)
        ddg = np.diagonal(dD, axis1=1, axis2=2)
        small = np.abs(dg) < 1e-6
        ambiguous = (np.abs(np.abs(dg) - 1e-6) <= ddg).any(axis=1)
        p = np.where(small, 1.0, 1.0 / np.where(small, 1.0, dg))
        dp = np.where(small, 0.0, ddg / np.where(small, 1.0, np.abs(dg)) + 2 * U)
        scale = np.ones((N, 6, 6))
        if by_column:
            scale[:, :, :3] = p[:, None, :3]
            rel = np.zeros((N, 6, 6)) + dp[:, None, :]
        else:
            scale[:, :, :3] = p[:, :, None]
            rel = np.zeros((N, 6, 6)) + dp[:, :, None]
        rel[:, :, 3:] = 0.0
        Dt = D * scale
        return Dt, dD * np.abs(scale) + rel * np.abs(Dt) + U * np.abs(Dt), p, dp, ambiguous

    def visc_beta(self, dens, beta, c_pass, by_column=False):
        """beta (N, 36 row-major) read back against the LU backward-error bound (Higham 9, 14.3), not against a float64
        inverse: with the column scaling undone (x_k = beta_k / p_k, k < 3), |Dt x_k - e_k| <= (|dDt| + 2 gamma_18
        |L||U|) |x_k| (+ the scaling's own error), |L||U| from a float64 partial-pivoting LU of Dt.  The gate: beta = 0
        exactly when |det| < 1e-6 (on the float32 LU) or a pivot is 0.  Returns (ratio, gate_violations, excluded, zero):
        excluded where the preconditioner switch or |det| lies within its bound of 1e-6; zero: beta = 0."""
        import scipy.linalg
        Dt, dDt, p, dp, amb = self.visc_matrix(dens, c_pass, by_column)
        N = self.N
        B = np.asarray(beta, np.float64).reshape(N, 6, 6)
        zero = ~B.any(axis=(1, 2))
        X = B.copy()
        X[:, :, :3] /= p[:, None, :3]
        gam = 18 * U / (1 - 18 * U)
        LU = np.zeros((N, 6, 6))
        det = np.zeros(N)
        det_b = np.full(N, np.inf)
        for k in range(N):
            P_, L_, U_ = scipy.linalg.lu(Dt[k])
            LU[k] = P_ @ (np.abs(L_) @ np.abs(U_))
            det[k] = np.linalg.det(Dt[k])
            if not Dt[k].any() and not dDt[k].any():   # no contact but itself: exactly singular
                det_b[k] = 0.0
            elif np.all(np.abs(np.diag(U_)) > 0):
                inv = np.linalg.inv(Dt[k])
                det_b[k] = 2 * abs(det[k]) * (np.abs(inv.T) * (dDt[k] + 2 * gam * LU[k])).sum()
        E = dDt + 2 * gam * LU
        res = np.abs(np.einsum("nrc,nck->nrk", Dt, X) - np.eye(6))
        bnd = np.einsum("nrc,nck->nrk", E, np.abs(X)) + \
            np.einsum("nrc,nck->nrk", np.abs(Dt), np.abs(X) * np.concatenate([dp[:, :3], np.zeros((N, 3))], 1)[:, None, :])
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(bnd > 0, res / bnd, np.where(res == 0, 0.0, np.inf)).max(axis=(1, 2))
        amb = amb | (np.abs(np.abs(det) - 1e-6) <= det_b)
        below = np.abs(det) + det_b < 1e-6
        violations = (zero & ~below & ~amb) | (~zero & below & ~amb)
        ratio = np.where(zero | amb, 0.0, ratio)
        return ratio, int(violations.sum()), amb, zero

    def visc_rates(self, dens, vel, acc, dt, scale, skip_adt=False):
        """The strain rate scale * sum_j m_j / (2 rho_i) S(grad W_ij, vv_j - vv_i) over the same fluid, vv = v + a dt as
        k_visc_vv forms it (dfsph_viscosity.rs:203-252): a Ref (N, 6).  scale: (1 - visc) for the target, 1 for the
        error.  skip_adt: vv = v."""
        sf, G, GA, GK = self._visc_grads(dens)
        v, a, dt = _f64(vel), _f64(acc), float(F(dt))
        vv = v + (0.0 if skip_adt else a * dt)
        vvA = np.abs(v) + (0.0 if skip_adt else np.abs(a) * dt)
        dv, dvA = vv[sf.j] - vv[sf.i], vvA[sf.j] + vvA[sf.i]

        def rate(g, d):
            x, y, z = g[:, 0], g[:, 1], g[:, 2]
            return np.stack([2 * d[:, 0] * x, 2 * d[:, 1] * y, 2 * d[:, 2] * z, d[:, 0] * y + d[:, 1] * x,
                             d[:, 0] * z + d[:, 2] * x, d[:, 1] * z + d[:, 2] * y], 1)
        N, s = self.N, abs(scale)
        return Ref(scale * _sum(N, sf.i, rate(G, dv)), s * _sum(N, sf.i, rate(GA, dvA)), s * _sum(N, sf.i, rate(GK, dvA)),
                   self._n(sf).astype(np.float64))

    def visc_accel(self, dens, beta, rate, rate_err, target, acc0, inv_dt, beta_i_for_j=False):
        """acc0 + sum_j G(grad W_ij)^T (u_i + u_j) m_j / 2 * m_i inv_dt over the same fluid (dfsph_viscosity.rs:254-289),
        u = beta (rate - target) / rho^2 with beta and target read back; rate: the float64 strain rate and rate_err its
        bound, carried through |beta|.  beta_i_for_j: u_j formed with beta_i."""
        sf, G, GA, GK = self._visc_grads(dens)
        N, rho = self.N, _f64(dens)
        B = np.asarray(beta, np.float64).reshape(N, 6, 6)
        err = rate - _f64(target)
        errA = np.abs(rate) + np.abs(_f64(target))
        u = np.einsum("nrk,nk->nr", B, err) / (rho * rho)[:, None]
        e_u = (np.einsum("nrk,nk->nr", np.abs(B), rate_err + 10 * U * errA)) / (rho * rho)[:, None]
        uA = np.einsum("nrk,nk->nr", np.abs(B), errA) / (rho * rho)[:, None]
        if beta_i_for_j:
            uj = np.einsum("nrk,nk->nr", B[sf.i], err[sf.j]) / (rho * rho)[sf.j][:, None]
        else:
            uj = u[sf.j]
        hm = self.mass[sf.j] / 2.0 * self.mass[sf.i] * float(F(inv_dt))
        c, cA, cE = (u[sf.i] + uj) * hm[:, None], (uA[sf.i] + uA[sf.j]) * hm[:, None], (e_u[sf.i] + e_u[sf.j]) * hm[:, None]
        tr = lambda m, w: np.einsum("nrk,nr->nk", m, w)  # noqa: E731
        Mt, MA, MK = self._mat6(G / (self.mass[sf.j] / (2.0 * rho[sf.i]))[:, None]), \
            self._mat6(GA / (self.mass[sf.j] / (2.0 * rho[sf.i]))[:, None]), self._mat6(GK / (self.mass[sf.j] / (2.0 * rho[sf.i]))[:, None])
        a0 = _f64(acc0)
        return Ref(a0 + _sum(N, sf.i, tr(Mt, c)), np.abs(a0) + _sum(N, sf.i, tr(MA, cA)),
                   _sum(N, sf.i, tr(MK, cA) + tr(MA, cE)), self._n(sf).astype(np.float64))

    def he2014_boundary_force(self, dens, gradc, cb, bvol, sign=-1.0):
        """He2014's reaction on boundary particles (he2014_surface_tension.rs:175): -f per contact.  sign: the sign of f."""
        fb, (b, bA, bK) = self._he2014_boundary_terms(dens, gradc, cb, bvol)
        return self._on_boundary(fb, sign * b, bA, bK)


class Becker:
    """Becker2009Elasticity's passes (becker2009_elasticity.rs:84-334) over the rest contacts: the same-fluid contacts of
    the rest positions Q (self included), always with the cubic spline.  Particles are in the fluids' original order, fluids
    concatenated; fid: the fluid of each, mass: float32 masses.  rest: other contacts to use (a kernel that recaptures its
    lists).  rows: rest contacts of these particles only (contacts_rows; the passes are exact at the rows)."""

    def __init__(self, h, Q, fid, mass, young, poisson, nonlinear, rest=None, rows=None):
        self.h = float(F(h))
        self.N, self.mass, self.nonlinear, self.fid = len(Q), _f64(mass), nonlinear, np.asarray(fid)
        same = lambda i, j: fid[i] == fid[j]  # noqa: E731
        if rest is None:
            rest = contacts(Q, Q, self.h, same, same=True) if rows is None else contacts_rows(Q, Q, self.h, same, rows)
        self.rest = rest
        r = self.rest
        E, nu, one, two = F(young), F(poisson), F(1.0), F(2.0)   # elasticity_coefficients :15-25, in float32 as solved
        self.d0 = float(F((E * (one - nu)) / ((one + nu) * (one - two * nu))))
        self.d1 = float(F((E * nu) / ((one + nu) * (one - two * nu))))
        self.d2 = float(F((E * (one - two * nu)) / (two * (one + nu) * (one - two * nu))))
        self.w, _, self.we = kernel(0, "w", r.r, self.h)
        g, _, ge = kernel(0, "g", r.r, self.h)
        z = r.d2 <= grad_threshold(0, self.h)
        self.g, self.ge = np.where(z, 0.0, g), np.where(z, 0.0, ge)
        self.n = np.bincount(r.i, minlength=self.N).astype(np.float64)

    def volume_sum(self, per_contact=2.0, old=None):
        """old_i + sum_j 2 m_j W0_ij: the rest volume is m_i over it (:89-111; each contact adds to both ends, the self
        contact included).  per_contact: the factor (1: each contact counted once).  old: the rest volumes a re-capture
        starts from (Vec::resize keeps the leading old values; 0 for new particles)."""
        r, N = self.rest, self.N
        t = per_contact * self.mass[r.j] * self.w
        o = np.zeros(N) if old is None else _f64(old)
        return Ref(o + _sum(N, r.i, t), np.abs(o) + _sum(N, r.i, np.abs(t)), _sum(N, r.i, per_contact * self.mass[r.j] * self.we),
                   self.n + (old is not None))

    def _pq(self, P):
        """Per rest contact p = x_j - x_i (current, float64 of float32) and q = x0_j - x0_i."""
        P = _f64(P)
        return P[self.rest.j] - P[self.rest.i], -self.rest.x

    def apq(self, P, c_pass):
        """A_pq = sum_j p_j q_j^T W0_ij m_j (:115-137) in float64 at the current positions P, and the bound of each entry
        of its float32 evaluation: (N, 3, 3) each."""
        r, N = self.rest, self.N
        p, q = self._pq(P)
        cw = self.w * self.mass[r.j]
        pq = p[:, :, None] * q[:, None, :]
        A = np.stack([_sum(N, r.i, pq[:, a, :] * cw[:, None]) for a in range(3)], axis=1)
        dA = np.stack([(self.n + c_pass)[:, None] * U * _sum(N, r.i, np.abs(pq[:, a, :]) * cw[:, None]) +
                       _sum(N, r.i, np.abs(pq[:, a, :]) * (self.mass[r.j] * self.we)[:, None]) for a in range(3)], axis=1)
        return A, dA

    def rotation(self, P, R_hat, R_prev, c_pass):
        """(ratio, orthonormality ratio, excluded, reference, iterations) of the float32 rotations R_hat (N, 3, 3) at the
        current positions P.  The reference is from_matrix_eps (rotation_from_matrix_eps) restated in float64 and run from
        the same warm start R_prev (the previous step's float32 rotations) on A_pq formed in float64.  The bound is the polar
        factor's perturbation bound 2 |dA|_F / (s2 + s3) (s3 negative when det A < 0), dA the float32 A_pq's error, plus
        the iteration's stopping test |axis / denom| <= eps (a residual angle of about eps (s1 + s2 + s3) / (s2 + s3)) and
        R_hat's own departure from orthonormality.  Excluded: particles where that bound exceeds 0.05 (s2 + s3 too small for
        the rotation to be determined), and those whose float64 run needs all 20 iterations."""
        A, dA = self.apq(P, c_pass)
        R, iters = from_matrix_eps(A, np.asarray(R_prev, np.float64))
        s = np.linalg.svd(A, compute_uv=False)
        d = np.sign(np.linalg.det(A))
        gap = s[:, 1] + d * s[:, 2]
        gs = np.where(gap > 0, gap, 1.0)
        ortho = np.abs(np.einsum("nki,nkj->nij", R_hat, R_hat) - np.eye(3)).max(axis=(1, 2))
        bound = 2 * np.sqrt((dA * dA).sum(axis=(1, 2))) / gs + (EPS32 + 8 * U) * (s[:, 0] + s[:, 1] + d * s[:, 2]) / gs + \
            C_EL_ORTHO * U
        excluded = (gap <= 0) | (bound > 0.05) | (iters >= 20)
        err = np.abs(np.asarray(R_hat, np.float64) - R).max(axis=(1, 2))
        return np.where(excluded, 0.0, err / bound), ortho / (C_EL_ORTHO * U), excluded, R, iters

    @staticmethod
    def polar(A):
        """The rotation of A's polar decomposition (SVD, det-corrected): the maximiser of tr(R^T A)."""
        u, _, vt = np.linalg.svd(A)
        d = np.sign(np.linalg.det(u @ vt))
        return (u * np.stack([np.ones(len(A)), np.ones(len(A)), d], axis=1)[:, None, :]) @ vt

    def grad_tr(self, P, R_hat, vol0):
        """deformation_gradient_tr_i = sum_j (vol0_j grad W0_ij) (R_i^T p_j - q_j)^T (:139-180), fed R_hat and vol0 read back
        (N, 3, 3), row-major.  R^T p - q cancels, so its absolute evaluation |R|^T |p| + |q| is carried in A."""
        r, N = self.rest, self.N
        R = np.asarray(R_hat, np.float64)
        v0 = _f64(vol0)
        p, q = self._pq(P)
        uu = np.einsum("nki,nk->ni", R[r.i], p) - q
        uA = np.einsum("nki,nk->ni", np.abs(R[r.i]), np.abs(p)) + np.abs(q)
        a = (self.g * v0[r.j])[:, None] * r.x
        aA = np.abs(a)
        aK = (self.ge * np.abs(v0[r.j]))[:, None] * np.abs(r.x)
        t = lambda x, y: np.stack([_sum(N, r.i, x[:, k, None] * y).reshape(N, 3) for k in range(3)], axis=1).reshape(N, 9)  # noqa: E731
        return Ref(t(a, uu), t(aA, uA), t(aK, uA), self.n)

    def stress(self, G):
        """Stress (x y z w a b) from deformation_gradient_tr G (N, 3, 3) read back (:182-262): linear, with the diagonal of G
        as the strain, or nonlinear, with J J^T - I, J = G + I; k = 0.564.  Ref with A the absolute evaluation (no sum)."""
        G = np.asarray(G, np.float64)
        k, d0, d1, d2 = float(F(0.564)), self.d0, self.d1, self.d2
        I = np.eye(3)
        if self.nonlinear:
            J, JA = G + I, np.abs(G) + I
            M, MA = J @ J.transpose(0, 2, 1), JA @ JA.transpose(0, 2, 1)
            e, eA = np.diagonal(M, axis1=1, axis2=2) - 1.0, np.diagonal(MA, axis1=1, axis2=2) + 1.0
            off, offA, ks = (M[:, 1, 0], M[:, 2, 0], M[:, 2, 1]), (MA[:, 1, 0], MA[:, 2, 0], MA[:, 2, 1]), k
        else:
            e, eA = np.diagonal(G, axis1=1, axis2=2), np.abs(np.diagonal(G, axis1=1, axis2=2))
            off = (G[:, 1, 0] + G[:, 0, 1], G[:, 2, 0] + G[:, 0, 2], G[:, 1, 2] + G[:, 2, 1])
            offA = (np.abs(G[:, 1, 0]) + np.abs(G[:, 0, 1]), np.abs(G[:, 2, 0]) + np.abs(G[:, 0, 2]),
                    np.abs(G[:, 1, 2]) + np.abs(G[:, 2, 1]))
            ks = 1.0
        D = np.array([[d0, d1, d1], [d1, d0, d1], [d1, d1, d0]])
        val = np.concatenate([(e @ D.T) * ks, np.stack(off, 1) * k * d2], axis=1)
        A = np.concatenate([(eA @ np.abs(D).T) * ks, np.stack(offA, 1) * k * abs(d2)], axis=1)
        N = len(G)
        return Ref(val, A, np.zeros_like(A), np.zeros(N))

    def force(self, S, G, R_hat, vol0, r_i_for_r_j=False, g_i_for_g_j=False):
        """The acceleration sum_j 0.5 (R_j f_ij - R_i f_ji) / m_i (:268-334), fed the stress S (N, 6), G, R_hat (N, 3, 3) and
        vol0 read back; f_ji = (s_i d_ij [+ G_i s_i d_ij]) (-vol0_i) with d_ij = grad W0_ij vol0_j, and f_ij likewise with
        j's stress, G and d_ji = -grad W0_ij vol0_i.  r_i_for_r_j / g_i_for_g_j: R_i / G_i in place of R_j / G_j."""
        r, N = self.rest, self.N
        S, G, R, v0 = np.asarray(S, np.float64), np.asarray(G, np.float64), np.asarray(R_hat, np.float64), _f64(vol0)
        sym = S[:, [0, 3, 4, 3, 1, 5, 4, 5, 2]].reshape(N, 3, 3)
        Rj = R[r.i] if r_i_for_r_j else R[r.j]
        Gj = G[r.i] if g_i_for_g_j else G[r.j]

        def terms(gk, absolute):
            ab = np.abs if absolute else (lambda x: x)
            grad = gk[:, None] * (np.abs(r.x) if absolute else r.x)
            d_ij, d_ji = grad * ab(v0[r.j])[:, None], grad * (ab(v0[r.i]) if absolute else -v0[r.i])[:, None]
            sd_ij = np.einsum("nab,nb->na", ab(sym[r.i]), d_ij)
            sd_ji = np.einsum("nab,nb->na", ab(sym[r.j]), d_ji)
            if self.nonlinear:
                sd_ij = sd_ij + np.einsum("nab,nb->na", ab(G[r.i]), sd_ij)
                sd_ji = sd_ji + np.einsum("nab,nb->na", ab(Gj), sd_ji)
            f_ji = sd_ij * (ab(v0[r.i]) if absolute else -v0[r.i])[:, None]
            f_ij = sd_ji * (ab(v0[r.j]) if absolute else -v0[r.j])[:, None]
            a, b = np.einsum("nab,nb->na", ab(Rj), f_ij), np.einsum("nab,nb->na", ab(R[r.i]), f_ji)
            return ((a + b) if absolute else (a - b)) * (0.5 / self.mass[r.i])[:, None]

        t, tA, tK = terms(self.g, False), terms(np.abs(self.g), True), terms(self.ge, True)
        return Ref(_sum(N, r.i, t), _sum(N, r.i, tA), _sum(N, r.i, tK), self.n)


def _tree_levels(threads):
    """Additions on the longest path of block_sum (sph_kernels.cuh) over `threads` lanes: warp_sum's five butterfly levels,
    then warp_sum again over the ceil(threads / 32) warp sums, padded with zeros (adding 0 is exact, so only
    ceil(log2(warps)) of those five levels round)."""
    warps = -(-threads // 32)
    return 5 + int(np.ceil(np.log2(warps))) if warps > 1 else 5


def structural_depth(n, block, second):
    """The depth D of the float32 loop-error reduction of n terms, derived from the kernels:
      1. each pass block of `block` threads sums one term per thread with block_sum's fixed tree (reduce_error in
         sph_passes.cuh; the neighbour search's fused first evaluation sums each warp, then the last warp to arrive sums
         the NBR_T / 32 warp sums, the same shape): _tree_levels(block) roundings on any term's path;
      2. the block that sums the nblk = ceil(n / block) partials (a pass's last block by ticket, blockDim = PASS_T, or
         k_reduce_partials with 256 threads) runs thread t over partials t, t + T, t + 2T, ... into s = 0: at most
         ceil(nblk / T) terms, of which the first is added to 0 exactly, so ceil(nblk / T) - 1 roundings;
      3. block_sum over those T per-thread sums: _tree_levels(T) roundings.
    Every term's path through this tree has at most D = (1) + (2) + (3) roundings of relative size u, so the float32
    result differs from the exact sum by at most gamma_D sum |e|, gamma_D = D u / (1 - D u) (Higham, Accuracy and
    Stability, 4.2), whatever the values.  At C3 (n = 10 077 696, 78 732 blocks of 128) D = 7 + 615 + 7 = 629 for a
    pass's last block and 7 + 307 + 8 = 322 for k_reduce_partials, against the n + 4 of the any-order bound.
    Sensitivity: losing every partial past block 65 535 (16.8 % of the terms at C3) is about 4000 times this bound;
    losing one block of 128 terms (1.3e-5 of the sum) lies below it (gamma_629 = 3.7e-5), so no honest bound can see that at
    this size: the small scenes' error_drops_last_block mutant covers it."""
    nblk = -(-max(n, 1) // block)
    return _tree_levels(block) + max(-(-nblk // second) - 1, 0) + _tree_levels(second)


def emulate_reduction(e, block, second):
    """The float32 value of the reduction structural_depth describes, emulated in numpy: e (float32, n terms) in blocks
    of `block`, warp butterflies, the warp-sum tree, the strided per-thread sums of the partials and the final block tree.
    Returns (float32 result, float32 partials)."""
    e = np.asarray(e, F)
    nblk = -(-len(e) // block)
    x = np.zeros(nblk * block, F)
    x[:len(e)] = e
    part = _block_sum(x.reshape(nblk, block))
    T = second
    m = -(-nblk // T)
    y = np.zeros(m * T, F)
    y[:nblk] = part
    y = y.reshape(m, T)
    s = np.zeros(T, F)
    for k in range(m):
        s = (s + y[k]).astype(F)
    return _block_sum(s[None, :])[0], part


def _block_sum(x):
    """block_sum over the last axis (float32): warp_sum per 32 lanes, then warp_sum over the warp sums padded to 32."""
    rows, t = x.shape
    w = -(-t // 32)
    v = np.zeros((rows, w * 32), F)
    v[:, :t] = x
    v = _warp_sum(v.reshape(rows, w, 32))
    pad = np.zeros((rows, 32), F)
    pad[:, :w] = v[:, :, 0]
    return _warp_sum(pad)[:, 0]


def _warp_sum(v):
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lane ^ o]).astype(F)
    return v


def from_matrix_eps(A, R0, eps=EPS32, max_iter=20):
    """nalgebra 0.33 Rotation3::from_matrix_eps (Mueller et al. 2016) in float64, vectorised over (N, 3, 3): from R0, while
    |aa| > eps with aa = sum_k r_k x a_k / (|sum_k r_k . a_k| + eps) (columns), R <- rot(aa) R.  Returns (R, iterations),
    iterations = 20 where the loop did not stop by itself."""
    R = R0.copy()
    iters = np.zeros(len(A), np.int64)
    active = np.ones(len(A), bool)
    for _ in range(max_iter):
        axis = sum(np.cross(R[:, :, k], A[:, :, k]) for k in range(3))
        denom = sum((R[:, :, k] * A[:, :, k]).sum(1) for k in range(3))
        aa = axis / (np.abs(denom) + eps)[:, None]
        active &= (aa * aa).sum(1) > eps * eps
        if not active.any():
            break
        ang = np.linalg.norm(aa, axis=1)
        u = aa / np.where(ang > 0, ang, 1.0)[:, None]
        K = np.zeros((len(A), 3, 3))
        K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -u[:, 2], u[:, 1], -u[:, 0]
        K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = u[:, 2], -u[:, 1], u[:, 0]
        D = np.eye(3) + np.sin(ang)[:, None, None] * K + (1 - np.cos(ang))[:, None, None] * (K @ K)
        R[active] = (D @ R)[active]
        iters[active] += 1
    return R, iters


def _f64(a):
    return np.asarray(a, F).astype(np.float64)


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
