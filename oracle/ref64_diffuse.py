"""Float64 restatement of the diffuse-particle update (include/sph.h sph_world_update_diffuse, DESIGN.md section 16).

TEST INFRASTRUCTURE ONLY.
  - `hash32` / `unit`: the counter-based hash of salva_b200/csrc/sph_hash.h on numpy uint32, bit for bit.
  - `normals64`, `potentials64`: n, I_ta, I_wc (kappa and its gate) and E_k per fluid particle in float64, each with the bound
    its float32 evaluation must meet ((n + c) u A + K, as ref64.py bounds a gather pass), and the pairs or gates whose
    decision lies within rounding of its threshold.
  - `counts32`: step 3's clamp and rounding in float32 numpy, operation by operation, from float32 potentials.
  - `binned_order`, `emit64`: the emission order and the cylinder sampling (Duff et al. 2017's basis) in float64.
  - `advect64`: classification and advection of diffuse particles against the fluid, with the bound of v~.
The keyword arguments named `mutant` inject the bugs the tests must catch.
"""
import numpy as np
from scipy.spatial import cKDTree

from oracle.ref64 import U, f32_d2, kernel
from oracle import ref64_surface as S

F = np.float32
M32 = np.uint64(0xFFFFFFFF)
SPRAY, FOAM, BUBBLE = 0, 1, 2
C_TA = 24    # per term: v_ij 1 + |v_ij| 4, the dot 5, / (|v| r) 2, 1 - c 1, W~ 2, products 2, fma 0; margin 9
C_WC = 16    # per term: the dot 5, 1 - nn 1, W~ 2, fma 0; margin 8
C_VT = 16    # v~: W (kernel normalisation 11 carried by C_NORM-like margin) + fma 0 + sums; margin
GATE = 0.6


# ---- hash ------------------------------------------------------------------------------------------------------------------
def mix32(x):
    x = np.asarray(x, np.uint64) & M32
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & M32
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & M32
    x ^= x >> np.uint64(16)
    return x


def hash32(seed, counter, slot, ident, k, stream):
    u = lambda a: np.asarray(a, np.uint64) & M32  # noqa: E731
    h = mix32(u(seed) ^ np.uint64(0x9E3779B9))
    h = mix32(h ^ u(counter))
    h = mix32(h ^ ((u(slot) << np.uint64(2)) | u(stream)))
    h = mix32(h ^ u(ident))
    return mix32(h ^ u(k)).astype(np.uint32)


def unit(h):
    """(h >> 8) 2^-24 as float32 (exact)."""
    return ((np.asarray(h, np.uint32) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24).astype(F)


# ---- clamp and counts ------------------------------------------------------------------------------------------------------
def phi(I, lo, hi):
    """Phi(I, lo, hi) = (min(I, hi) - min(I, lo)) / (hi - lo) in float64."""
    I = np.asarray(I, np.float64)
    return (np.minimum(I, hi) - np.minimum(I, lo)) / (hi - lo)


def _min32(a, b):
    return np.where(b < a, b, a).astype(F)


def phi32(I, lo, hi):
    I, lo, hi = np.asarray(I, F), F(lo), F(hi)
    return ((_min32(I, hi) - _min32(I, lo)).astype(F) / F(hi - lo)).astype(F)


def counts32(ta, wc, ek, slots, ids, d, dt, counter):
    """n_d of include/sph.h step 3 in float32 from the float32 potentials (uint64 counts)."""
    pta, pwc, pk = phi32(ta, d["ta_min"], d["ta_max"]), phi32(wc, d["wc_min"], d["wc_max"]), phi32(ek, d["k_min"], d["k_max"])
    u = unit(hash32(d["seed"], counter, slots, ids, 0, 0))
    s = ((F(d["k_ta"]) * pta).astype(F) + (F(d["k_wc"]) * pwc).astype(F)).astype(F)
    e = ((((pk * s).astype(F)) * F(dt)).astype(F) + u).astype(F)
    with np.errstate(invalid="ignore"):
        return np.where(e >= F(1), np.where(e >= F(4294967296.0), 0xFFFFFFFF, np.floor(np.where(np.isfinite(e), e, 0))), 0).astype(np.uint64)


# ---- pairs -------------------------------------------------------------------------------------------------------------------
def pairs(P, Q, h):
    """(i, j) with the unfused float32 test |P_i - Q_j|^2 <= h^2 (rows of P against rows of Q), i ascending."""
    P, Q = np.asarray(P, F), np.asarray(Q, F)
    if not len(P) or not len(Q):
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    ok = np.all(np.isfinite(P), axis=1)
    lists = cKDTree(Q.astype(np.float64)).query_ball_point(np.where(ok[:, None], P, 0).astype(np.float64), h * (1 + 1e-5))
    cnt = np.fromiter((len(l) if o else 0 for l, o in zip(lists, ok)), np.int64, len(lists))
    i = np.repeat(np.arange(len(P)), cnt)
    j = np.concatenate([np.asarray(l, np.int64) for l, o in zip(lists, ok) if o and len(l)] or [np.zeros(0, np.int64)])
    keep = f32_d2(P[i], Q[j]) <= F(F(h) * F(h))
    return i[keep], j[keep]


# ---- normals and potentials ------------------------------------------------------------------------------------------------
def normals64(x, vol, h, kind_g=0):
    """(n, bound of |n - n64| per particle): -grad phi / |grad phi| at the particles; bound 2 where the gradient is not
    resolved (|grad phi| <= 1000 times its bound)."""
    n, m, gb = S.normals64(x, vol, np.asarray(x, F), h, kind_g)
    e = np.where(m > 1000.0 * gb, 2.0 * np.sqrt(3.0) * gb / np.where(m > 0, m, 1.0) + 1e-6, 2.0)
    return n, e


def potentials64(x, v, vol, rho0, n64, ne, h, mutant=None):
    """Per fluid particle: dict of ta, ta_b, kap (the wave-crest sum before the gate), kap_b, gate (v^ . n), gate_b, wc (the
    gated value with the gate decided in float64), ek, ek_b."""
    x, v = np.asarray(x, F).astype(np.float64), np.asarray(v, F).astype(np.float64)
    N = len(x)
    vol = np.broadcast_to(np.asarray(vol, F).astype(np.float64), (N,))
    rho0 = np.broadcast_to(np.asarray(rho0, F).astype(np.float64), (N,))
    i, j = pairs(x.astype(F), x.astype(F), h)
    xij, vij = x[i] - x[j], v[i] - v[j]
    r = np.sqrt((xij * xij).sum(1))
    vn = np.sqrt((vij * vij).sum(1))
    wt = np.exp(-r) if mutant == "W" else 1.0 - r / h  # the mutant: a smooth kernel in place of W~
    ok = (r > 0) & (vn > 0)
    c = np.where(ok, (vij * xij).sum(1) / np.where(ok, vn * r, 1.0), 0.0)
    t_ta = np.where(ok, vn * (1.0 - c) * wt, 0.0)
    a_ta = np.where(ok, vn * (1.0 + np.abs(c)) * (1.0 + r / h), 0.0)
    side = (xij * n64[i]).sum(1)
    if mutant == "convex":
        side = -side
    amb = np.abs(side) <= r * (ne[i] + 8 * U) + 1e-12
    nn = (n64[i] * n64[j]).sum(1)
    t_wc = np.where(side > 0, (1.0 - nn) * wt, 0.0)
    e_wc = np.where(side > 0, (ne[i] + ne[j]) * wt, 0.0) + np.where(amb, (np.abs(1.0 - nn) + ne[i] + ne[j]) * wt, 0.0)
    a_wc = np.where(side > 0, (1.0 + np.abs(nn)) * (1.0 + r / h), 0.0)
    cnt = np.bincount(i, minlength=N)
    ta = np.bincount(i, t_ta, N)
    kap = np.bincount(i, t_wc, N)
    ta_b = (cnt + C_TA) * U * np.bincount(i, a_ta, N)
    kap_b = (cnt + C_WC) * U * np.bincount(i, a_wc, N) + np.bincount(i, e_wc, N)
    vm = np.sqrt((v * v).sum(1))
    gate = np.where(vm > 0, (v * n64).sum(1) / np.where(vm > 0, vm, 1.0), 0.0)
    gate_b = ne + 8 * U
    wc = kap if mutant == "no_gate" else np.where(gate >= GATE, kap, 0.0)
    ek = 0.5 * vol * rho0 * (v * v).sum(1)
    return dict(ta=ta, ta_b=ta_b, kap=kap, kap_b=kap_b, gate=gate, gate_b=gate_b, wc=wc, ek=ek, ek_b=8 * U * ek, n=cnt)


# ---- emission ----------------------------------------------------------------------------------------------------------------
def cells(x, h):
    """floor(x / h) with the float32 division, per axis (int64)."""
    return np.floor((np.asarray(x, F) / F(h)).astype(F)).astype(np.int64)


def binned_order(x, slots, ids, h):
    """Rows of the finite positions in binned order: cell (x, y, z major to minor), then (fluid slot, id)."""
    x = np.asarray(x, F)
    fin = np.nonzero(np.all(np.isfinite(x), axis=1))[0]
    c = cells(x[fin], h)
    o = np.lexsort((np.asarray(ids)[fin], np.asarray(slots)[fin], c[:, 2], c[:, 1], c[:, 0]))
    return fin[o]


def basis(nv):
    """Duff et al. 2017: e1, e2 orthonormal to the unit vectors nv [n, 3] (float64)."""
    nv = np.asarray(nv, np.float64)
    s = np.where(np.signbit(nv[:, 2]), -1.0, 1.0)
    a = -1.0 / (s + nv[:, 2])
    b = nv[:, 0] * nv[:, 1] * a
    e1 = np.stack([1.0 + s * nv[:, 0] ** 2 * a, s * b, -s * nv[:, 0]], 1)
    e2 = np.stack([b, s + nv[:, 1] ** 2 * a, -nv[:, 1]], 1)
    return e1, e2


def emit64(xf, vf, slots, ids, counts, d, dt, counter, rp, room=None, mutant=None):
    """The emitted particles (x, v, bound per component) of the fluid rows given in emission order with their counts,
    cut after `room` particles."""
    xf, vf = np.asarray(xf, F).astype(np.float64), np.asarray(vf, F).astype(np.float64)
    counts = np.asarray(counts, np.int64)
    total = int(counts.sum())
    if room is not None:
        total = min(total, int(room) + (1 if mutant == "cut" else 0))
    rows = np.repeat(np.arange(len(counts)), counts)[:total]
    k = (np.arange(total) - np.repeat(np.cumsum(counts) - counts, counts)[:total]).astype(np.uint64)
    sl, idv = np.asarray(slots, np.uint64)[rows], np.asarray(ids, np.uint64)[rows]
    X = [unit(hash32(d["seed"], counter, sl, idv, k, s)).astype(np.float64) for s in (1, 2, 3)]
    sp = np.sqrt((vf[rows] ** 2).sum(1))
    nv = np.where(sp[:, None] > 0, vf[rows] / np.where(sp > 0, sp, 1.0)[:, None], 0.0)
    e1, e2 = basis(nv)
    r = rp * np.sqrt(X[0])
    th = 2.0 * np.pi * X[1]
    o = (r * np.cos(th))[:, None] * e1 + (r * np.sin(th))[:, None] * e2
    x = xf[rows] + o + (X[2] * dt)[:, None] * vf[rows]
    v = vf[rows] + o
    # sin / cos (a few ulp) and the float32 basis and sums: relative to the magnitudes involved
    bx = 64 * U * (np.abs(xf[rows]) + rp + np.abs(vf[rows]) * dt)
    bv = 64 * U * (np.abs(vf[rows]) + rp)
    return x, v, bx, bv, rows


# ---- classification and advection -------------------------------------------------------------------------------------------
def advect64(xd, vd, life, xf, vf, h, d, dt, g, kind_w=0, mutant=None):
    """(x, v, life, kind, n_n, bound of x, bound of v, keep) of every diffuse particle after one advection."""
    xd, vd = np.asarray(xd, F), np.asarray(vd, F).astype(np.float64)
    life = np.asarray(life, F).astype(np.float64)
    g = np.asarray(g, np.float64)
    n = len(xd)
    i, j = pairs(xd, xf, h)
    r = np.sqrt(((xd[i].astype(np.float64) - np.asarray(xf, F)[j].astype(np.float64)) ** 2).sum(1))
    W, Wa, Wk = kernel(kind_w, "w", r, h)
    vj = np.asarray(vf, F).astype(np.float64)[j]
    nn = np.bincount(i, minlength=n)
    sw = np.bincount(i, W, n)
    num = np.stack([np.bincount(i, W * vj[:, a], n) for a in range(3)], 1)
    eD = (nn + 14) * U * np.bincount(i, Wa, n) + np.bincount(i, Wk, n)
    eN = np.stack([(nn + 14) * U * np.bincount(i, Wa * np.abs(vj[:, a]), n) + np.bincount(i, Wk * np.abs(vj[:, a]), n) for a in range(3)], 1)
    vt = np.where(sw[:, None] > 0, num / np.where(sw > 0, sw, 1.0)[:, None], 0.0)
    evt = np.where(sw[:, None] > 0, (eN + np.abs(vt) * eD[:, None]) / np.where(sw > 0, sw, 1.0)[:, None] + 2 * U * np.abs(vt), 0.0)
    if mutant == "inclusive":  # the classification thresholds counted inclusively
        kind = np.where(nn <= d["spray_below"], SPRAY, np.where(nn >= d["bubble_above"], BUBBLE, FOAM))
    else:
        kind = np.where(nn < d["spray_below"], SPRAY, np.where(nn > d["bubble_above"], BUBBLE, FOAM))
    x0 = xd.astype(np.float64)
    v = np.where((kind == SPRAY)[:, None], vd + dt * g, np.where((kind == BUBBLE)[:, None], vd - dt * d["k_b"] * g + d["k_d"] * (vt - vd), vt))
    ev = np.where((kind == SPRAY)[:, None], 2 * U * (np.abs(vd) + dt * np.abs(g)),
                  np.where((kind == BUBBLE)[:, None], d["k_d"] * evt + 6 * U * (np.abs(vd) + dt * d["k_b"] * np.abs(g) + d["k_d"] * np.abs(vt - vd)), evt))
    x = x0 + dt * v
    ex = dt * ev + 3 * U * (np.abs(x0) + dt * np.abs(v))
    ages = np.ones(n, bool) if mutant == "all_age" else kind == FOAM
    life = np.where(ages, life - dt, life)
    lo, hi = np.asarray(d["lo"], np.float64), np.asarray(d["hi"], np.float64)
    with np.errstate(invalid="ignore"):
        inside = np.all((lo <= x) & (x < hi), axis=1)
    keep = inside & ~((kind == FOAM) & ~(life > 0))
    return dict(x=x, v=v, life=life, kind=kind, nn=nn, ex=ex, ev=ev, keep=keep)
