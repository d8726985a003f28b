"""Float64 restatement of the anisotropic surface kernels (Yu & Turk 2013; include/sph.h
sph_world_extract_surface_anisotropic, DESIGN.md section 17), with the bounds their float32 evaluation must meet.

TEST INFRASTRUCTURE ONLY.
  - `ellipsoids64`: per particle the neighbours (the step's unfused float32 pair test), the centre x_bar, the covariance's
    eigen-decomposition, the radii and the shape matrix M = sum_k a_k^2 e_k e_k^T, all in float64 from the float32
    positions, with a bound for the centre and for M (derived below).  M is compared rather than the axes: it has no sign
    or eigenvector ambiguity.
  - `field64`: phi = sum_i V_i W_i at float32 points from given ellipsoid rows (the device's own), with its bound.
  - `grad64` / `normals64`: grad phi and -grad phi / |grad phi| from given ellipsoid rows, with the bound of grad phi.
  - `emulate32`: a float32 evaluation of the ellipsoid rule in numpy (running sums, cyclic Jacobi, the radii), for checking
    the bounds against a float32 evaluation without a GPU.  It is not the device's operation sequence: it rounds where the
    device fuses (fma), divides where it takes rsqrt, and always runs 8 sweeps; the device tests check the device itself.
Keyword arguments named after a bug inject that bug (the mutants the tests must catch).

Bounds (u = 2^-24, T = N_i + 1 summed terms, the sums taken relative to x_i so every offset |d| <= h):
  each weight w = 1 - (fl(sqrt(d2)) / h)^3 is off by at most 15 u (d2 3 u, sqrt and / 1 u each, the cube 2 u, the
  difference 1 u); a running float32 sum of T terms is off by at most T u sum |terms|.  So
    E_w  = T u (sum w + 16),  E_m1 = T u (sum w |d| + 20 h)                (sum w, and each component of sum w d)
    |dm| <= (E_m1 + |m| E_w) / sum w + u |m|,  m = x^w - x_i,
    |d x_bar| <= lambda |dm| + u |x_bar|                                       (the fma lambda m + x_i)
  and with E_q = T u (sum w |d|^2 + 24 h^2) for each entry of sum w d d^T,
    |dC_ab| <= (E_q + |q_ab| E_w / sum w) / sum w + 2 |m| |dm| + 3 u (|q_ab| / sum w + |m|^2),
  plus the Jacobi sweeps' backward error, at most 100 u ||C||_F.  M = h^2 f(C / s1), f(s) = max(s, 1 / k_r)^2 applied to
  the eigenvalues; f is Lipschitz with constant 2 (1 + rho) on [0, 1 + rho], rho = ||dC||_F / s1, and a Lipschitz scalar
  function is Lipschitz with the same constant on symmetric matrices in the Frobenius norm (Kittaneh 1985); C / s1 moves by
  at most 2 ||dC||_F / s1.  So ||dM||_F <= 4 (1 + rho) h^2 ||dC||_F / s1 + 200 u h^2, the last term the rounding of the radii
  and the eigenvectors' loss of orthonormality over at most 24 rotations.  The bound is stated where rho <= 0.1; where s1 is
  within ||dC|| of 0 the branch itself is ambiguous and the bound is infinite.
"""
import numpy as np
from scipy.spatial import cKDTree

from oracle.ref64 import U, _KINDS, f32_d2

F = np.float32


def neighbour_pairs(positions, h):
    """(i, j) over i != j with the float32 unfused test (dx*dx + dy*dy) + dz*dz <= h*h, finite positions only."""
    p = np.asarray(positions, F)
    ok = np.all(np.isfinite(p), axis=1)
    idx = np.nonzero(ok)[0]
    if not len(idx):
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    tree = cKDTree(p[idx].astype(np.float64))
    pr = tree.query_pairs(float(h) * (1.0 + 1e-5), output_type="ndarray")
    if not len(pr):
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    i, j = idx[pr[:, 0]], idx[pr[:, 1]]
    keep = f32_d2(p[i], p[j]) <= F(h) * F(h)
    i, j = i[keep], j[keep]
    return np.concatenate([i, j]), np.concatenate([j, i])


def ellipsoids64(positions, h, smoothing=0.9, max_ratio=1.0, isolated_radius=1.0, min_neighbours=6, *, sqrt_radii=False,
                 clamp_before_sort=False, weights_linear=False, count_self=False, swap_lambda=False):
    """Per particle: dict of centre [n, 3], e [n, 3, 3] (columns e1, e2, e3), a [n, 3], M [n, 3, 3], count N [n], the
    centre bound [n] (per component), the M bound [n] (Frobenius; inf where the branch is ambiguous) and aniso [n] (the
    anisotropic branch).  Non-finite positions: centre = position, a = 0."""
    p32 = np.asarray(positions, F)
    x = p32.astype(np.float64)
    n = len(x)
    h = float(F(h))
    lam, kr, kn = float(F(smoothing)), float(F(max_ratio)), float(F(isolated_radius))
    i, j = neighbour_pairs(p32, h)
    fin = np.all(np.isfinite(p32), axis=1)
    N = np.bincount(i, minlength=n).astype(np.int64)
    d = x[j] - x[i]
    r = np.sqrt((d * d).sum(axis=1))
    w = 1.0 - (r / h) if weights_linear else 1.0 - (r / h) ** 3
    sw = 1.0 + np.bincount(i, w, minlength=n)
    s1 = np.stack([np.bincount(i, w * d[:, a], minlength=n) for a in range(3)], axis=1)
    q = np.zeros((n, 3, 3))
    for a in range(3):
        for b in range(3):
            q[:, a, b] = np.bincount(i, w * d[:, a] * d[:, b], minlength=n)
    swd = np.bincount(i, w * r, minlength=n)
    swd2 = np.bincount(i, w * r * r, minlength=n)
    m = s1 / sw[:, None]
    lam_eff = 1.0 - lam if swap_lambda else lam
    centre = np.where(fin[:, None], x + lam_eff * m, x)
    C = q / sw[:, None, None] - m[:, :, None] * m[:, None, :]
    sig, V = np.linalg.eigh(np.where(fin[:, None, None], C, 0.0))  # ascending
    sig = np.maximum(sig, 0.0)
    order = np.argsort(-sig, axis=1, kind="stable")
    sig_s = np.take_along_axis(sig, order, axis=1)
    V_s = np.take_along_axis(V, order[:, None, :], axis=2)
    cnt = N + 1 if count_self else N
    aniso = fin & (cnt >= min_neighbours) & (sig_s[:, 0] > 0)
    s1v = np.where(sig_s[:, 0] > 0, sig_s[:, 0], 1.0)
    if clamp_before_sort:  # the clamp and the normalisation against eigh's first (smallest) eigenvalue
        first = np.where(sig[:, 0] > 0, sig[:, 0], s1v)
        a = h * np.maximum(sig_s, (first / kr)[:, None]) / first[:, None]
    else:
        a = h * np.maximum(sig_s / s1v[:, None], 1.0 / kr)
    if sqrt_radii:
        a = h * np.sqrt(np.maximum(sig_s, (s1v / kr)[:, None]) / s1v[:, None])
    e = np.where(aniso[:, None, None], V_s, np.eye(3)[None])
    a = np.where(aniso[:, None], a, float(F(kn * h)))
    a = np.where(fin[:, None], a, 0.0)
    M = np.einsum("nik,nk,njk->nij", e, a * a, e)

    # bounds (module docstring)
    T = (N + 1).astype(np.float64)
    mm = np.sqrt((m * m).sum(axis=1))
    Ew = T * U * (sw + 16.0)
    Em1 = T * U * (swd + 20.0 * h)
    dm = (Em1 + mm * Ew) / sw + U * mm
    cbound = 2.0 * (lam_eff * dm + U * np.abs(centre).max(axis=1)) + 1e-30
    Eq = T * U * (swd2 + 24.0 * h * h)
    qa = np.abs(q) / sw[:, None, None]
    dC = (Eq[:, None, None] + qa * (Ew / sw)[:, None, None]) / sw[:, None, None] + 2.0 * (mm * dm)[:, None, None] \
        + 3.0 * U * (qa + (mm * mm)[:, None, None])
    dCf = np.sqrt((dC * dC).sum(axis=(1, 2))) + 100.0 * U * np.sqrt((C * C).sum(axis=(1, 2)))
    rho = dCf / s1v
    mb = 4.0 * (1.0 + rho) * h * h * dCf / s1v + 200.0 * U * h * h
    mb = np.where(aniso, np.where(rho <= 0.1, mb, np.inf), 200.0 * U * h * h)
    mb = np.where(fin & ~aniso & (cnt >= min_neighbours) & (sig_s[:, 0] <= dCf), np.inf, mb)
    return dict(centre=centre, e=e, a=a, M=M, N=N, sigma=sig_s, centre_bound=cbound, M_bound=mb, aniso=aniso, finite=fin)


def shape_rows(centres, axes, volumes, h):
    """From the device's rows (centres [n, 3], axes [n, 3, 4] = (e_k, a_k)): h G [n, 3, 3], the scale V h^3 / (a1 a2 a3) [n]
    and max_k h / a_k [n], in float64; rows with a zero axis (non-finite positions) get scale 0."""
    ax = np.asarray(axes, np.float64)
    e, a = ax[:, :, :3], ax[:, :, 3]
    ok = np.all(a > 0, axis=1) & np.all(np.isfinite(np.asarray(centres, np.float64)), axis=1)
    ia = np.where(ok[:, None], h / np.where(a > 0, a, 1.0), 0.0)
    H = np.einsum("nki,nk,nkj->nij", e, ia, e)
    v = np.broadcast_to(np.asarray(volumes, F).astype(np.float64), (len(ax),))
    return H, np.where(ok, v * ia.prod(axis=1), 0.0), ia.max(axis=1, initial=0.0), ok


def _kernel(kind, which, r, h, eps):
    fn = _KINDS[kind]
    f, fa = fn(which, r, h)
    up, _ = fn(which, r * (1.0 + eps), h)
    dn, _ = fn(which, r * (1.0 - eps), h)
    return f, fa, np.maximum(np.abs(up - f), np.abs(dn - f)) + eps * fa


def _pairs(centres, ok, pts, h):
    c = np.asarray(centres, np.float64)
    idx = np.nonzero(ok)[0]
    p = np.asarray(pts, F).astype(np.float64)
    if not len(idx) or not len(p):
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    tree = cKDTree(c[idx])
    lists = tree.query_ball_point(p, h * (1.0 + 1e-5))
    cnt = np.fromiter((len(l) for l in lists), np.int64, len(lists))
    if not cnt.sum():
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.repeat(np.arange(len(p)), cnt), idx[np.concatenate([np.asarray(l, np.int64) for l in lists if len(l)])]


def field64(centres, axes, volumes, pts, h, kind=0, *, swap_G=False, drop_det=False):
    """(phi, bound) at the float32 points from the ellipsoid rows.  The relative error of |u| on the device is at most
    (6 k + 4) u, k = a1 / a3 (rows rounded into h G 4 u, d 1 u, u = h G d 2 u, |u|^2 3 u); the scale is off by 6 u."""
    h = float(F(h))
    H, s, ia, ok = shape_rows(centres, axes, volumes, h)
    if swap_G:  # h G^-1 / h^2 in place of h G: the semi-axes and their inverses swapped
        H = np.linalg.inv(np.where(ok[:, None, None], H, np.eye(3))) * 1.0
    if drop_det:
        s = np.where(ok, np.broadcast_to(np.asarray(volumes, F).astype(np.float64), (len(s),)), 0.0)
    p = np.asarray(pts, F).astype(np.float64)
    phi, A, K, n = np.zeros(len(p)), np.zeros(len(p)), np.zeros(len(p)), np.zeros(len(p))
    i, j = _pairs(centres, ok, p, h)
    if len(i):
        d = p[i] - np.asarray(centres, np.float64)[j]
        u = np.einsum("nab,nb->na", H[j], d)
        r = np.sqrt((u * u).sum(axis=1))
        ax = np.asarray(axes, np.float64)[:, :, 3]
        k = ax.max(axis=1) / np.where(ax.min(axis=1) > 0, ax.min(axis=1), 1.0)
        f, fa, kerr = _kernel(kind, "w", r, h, (6.0 * k[j] + 4.0) * U)
        np.add.at(phi, i, s[j] * f)
        np.add.at(A, i, s[j] * fa)
        np.add.at(K, i, s[j] * kerr)
        np.add.at(n, i, 1.0)
    return phi, (n + 9.0) * U * A + K


def grad64(centres, axes, volumes, pts, h, kind=0, *, drop_G=False):
    """(grad phi [n, 3], bound per component) at the float32 points: sum s h G W'(|u|) / |u| u."""
    h = float(F(h))
    H, s, ia, ok = shape_rows(centres, axes, volumes, h)
    p = np.asarray(pts, F).astype(np.float64)
    g, A, K, n = np.zeros((len(p), 3)), np.zeros(len(p)), np.zeros(len(p)), np.zeros(len(p))
    i, j = _pairs(centres, ok, p, h)
    if len(i):
        d = p[i] - np.asarray(centres, np.float64)[j]
        u = np.einsum("nab,nb->na", H[j], d)
        r = np.sqrt((u * u).sum(axis=1))
        ax = np.asarray(axes, np.float64)[:, :, 3]
        k = ax.max(axis=1) / np.where(ax.min(axis=1) > 0, ax.min(axis=1), 1.0)
        f, fa, kerr = _kernel(kind, "g", r, h, (6.0 * k[j] + 4.0) * U)
        f = np.where(r * r > float(np.finfo(F).eps) ** 2, f, 0.0)
        t = (s[j] * f)[:, None] * u
        contrib = t if drop_G else np.einsum("nab,nb->na", H[j], t)
        np.add.at(g, i, contrib)
        hn = ia[j]  # ||h G||_2
        np.add.at(A, i, s[j] * hn * fa * r)
        np.add.at(K, i, s[j] * hn * kerr * r)
        np.add.at(n, i, 1.0)
    return g, (n + 20.0) * U * A + K


def normals64(centres, axes, volumes, verts, h, kind=0, **mut):
    g, gb = grad64(centres, axes, volumes, verts, h, kind, **mut)
    m = np.sqrt((g * g).sum(axis=1))
    return np.where(m[:, None] > 0, -g / np.where(m > 0, m, 1.0)[:, None], 0.0), m, gb


# ---- float32 emulation of the device rule -------------------------------------------------------------------------------
def emulate32(positions, h, smoothing=0.9, max_ratio=1.0, isolated_radius=1.0, min_neighbours=6):
    """(centre [n, 3], M [n, 3, 3] in float64 from float32 e and a): the rule evaluated in float32 numpy, sums in neighbour
    order, 8 cyclic Jacobi sweeps (rotations (0,1), (0,2), (1,2)), the descending sort, the radii."""
    p = np.asarray(positions, F)
    n = len(p)
    h = F(h)
    i, j = neighbour_pairs(p, h)
    o = np.lexsort((j, i))
    i, j = i[o], j[o]
    sw = np.ones(n, F)
    m = np.zeros((n, 3), F)
    q = np.zeros((n, 6), F)
    cnt = np.bincount(i, minlength=n)
    start = np.concatenate([[0], np.cumsum(cnt)])
    for k in range(int(cnt.max(initial=0))):
        sel = np.nonzero(cnt > k)[0]
        jj = j[start[sel] + k]
        dd = (p[sel] - p[jj]).astype(F)
        d2 = ((dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]).astype(F)
        qq = (np.sqrt(d2).astype(F) / h).astype(F)
        wt = (F(1) - ((qq * qq).astype(F) * qq).astype(F)).astype(F)
        od = -dd
        sw[sel] = (sw[sel] + wt).astype(F)
        wd = (wt[:, None] * od).astype(F)
        m[sel] = (m[sel] + wd).astype(F)
        for e_, (a, b) in enumerate(((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2))):
            q[sel, e_] = (q[sel, e_] + (wd[:, a] * od[:, b]).astype(F)).astype(F)
    m = (m / sw[:, None]).astype(F)
    centre = (F(smoothing) * m + p).astype(F)
    A = np.zeros((n, 3, 3), F)
    for e_, (a, b) in enumerate(((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2))):
        A[:, a, b] = A[:, b, a] = ((q[:, e_] / sw).astype(F) - (m[:, a] * m[:, b]).astype(F)).astype(F)
    V = np.broadcast_to(np.eye(3, dtype=F), (n, 3, 3)).copy()
    for _ in range(8):
        for (pp, qq_) in ((0, 1), (0, 2), (1, 2)):
            apq = A[:, pp, qq_]
            nz = apq != 0
            den = np.where(nz, F(2) * apq, F(1)).astype(F)
            th = ((A[:, qq_, qq_] - A[:, pp, pp]).astype(F) / den).astype(F)
            at = np.abs(th)
            with np.errstate(over="ignore"):
                t = np.where(at > F(1e18), (F(0.5) / np.maximum(at, F(1e-30))).astype(F),
                             (F(1) / (at + np.sqrt((at * at + F(1)).astype(F))).astype(F)).astype(F))
            t = np.where(nz, np.copysign(t, th), F(0)).astype(F)
            c = (F(1) / np.sqrt((t * t + F(1)).astype(F))).astype(F)
            s = (t * c).astype(F)
            r_ = 3 - pp - qq_
            arp, arq = A[:, r_, pp].copy(), A[:, r_, qq_].copy()
            A[:, pp, pp] = (A[:, pp, pp] - (t * apq).astype(F)).astype(F)
            A[:, qq_, qq_] = (A[:, qq_, qq_] + (t * apq).astype(F)).astype(F)
            A[:, pp, qq_] = np.where(nz, F(0), A[:, pp, qq_])
            A[:, qq_, pp] = A[:, pp, qq_]
            A[:, r_, pp] = A[:, pp, r_] = ((c * arp).astype(F) - (s * arq).astype(F)).astype(F)
            A[:, r_, qq_] = A[:, qq_, r_] = ((s * arp).astype(F) + (c * arq).astype(F)).astype(F)
            vp, vq = V[:, :, pp].copy(), V[:, :, qq_].copy()
            V[:, :, pp] = ((c[:, None] * vp).astype(F) - (s[:, None] * vq).astype(F)).astype(F)
            V[:, :, qq_] = ((s[:, None] * vp).astype(F) + (c[:, None] * vq).astype(F)).astype(F)
    sg = np.maximum(np.stack([A[:, 0, 0], A[:, 1, 1], A[:, 2, 2]], axis=1), F(0))
    order = np.argsort(-sg, axis=1, kind="stable")
    sg = np.take_along_axis(sg, order, axis=1)
    V = np.take_along_axis(V, order[:, None, :], axis=2)
    aniso = (cnt >= min_neighbours) & (sg[:, 0] > 0)
    s1 = np.where(sg[:, 0] > 0, sg[:, 0], F(1))
    a = (h * np.maximum((sg / s1[:, None]).astype(F), (F(1) / F(max_ratio)).astype(F))).astype(F)
    a[:, 0] = h
    a = np.where(aniso[:, None], a, F(isolated_radius) * h).astype(F)
    V = np.where(aniso[:, None, None], V, np.eye(3, dtype=F)[None])
    e, a = V.astype(np.float64), a.astype(np.float64)
    return centre, np.einsum("nik,nk,njk->nij", e, a * a, e)
