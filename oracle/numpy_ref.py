"""Independent brute-force (O(n^2), dense-matrix) numpy restatement of salva3d's DFSPH step.

TEST INFRASTRUCTURE ONLY.  Purpose: a second, structurally different implementation of the same
reference formulas (SURVEY.md Appendix A) to pin oracle/oracle.cpp, because the reference ships no
golden vectors (PARITY UNPINNED upstream).  Dense all-pairs matrices replace the hash grid and the
contact lists, so a shared bug in neighbour search or list handling cannot hide.

Cites (reference src/): kernel/cubic_spline_kernel.rs:12-33,55-80; kernel/kernel.rs:18-24;
geometry/contacts.rs:254-400 (pair rule); solver/pressure/dfsph_solver.rs (all);
solver/viscosity/{xsph,artificial}_viscosity.rs; solver/surface_tension/akinci2013_surface_tension.rs.
"""
import numpy as np

F = np.float32
EPS = np.float32(1.1920929e-07)


def _w(r, h):
    sigma = F(8.0) / (F(np.pi) * h * h * h)
    q = r / h
    q2 = q * q
    a = F(1.0) + (q2 * q - q2) * F(6.0)
    t = F(1.0) - q
    b = t * t * t * F(2.0)
    return sigma * np.where(q <= F(0.5), a, np.where(q <= F(1.0), b, F(0.0))).astype(F)


def _dw(r, h):
    sigma = F(8.0) / (F(np.pi) * h * h * h)
    q = r / h
    a = (q * F(3.0) - F(2.0)) * q * F(6.0)
    t = F(1.0) - q
    b = -t * t * F(6.0)
    rhs = np.where((q > F(1.0)) | (q <= F(1.0e-5)), F(0.0), np.where(q <= F(0.5), a, b)).astype(F)
    return sigma * rhs / h


def _powi(x, n):
    r = np.ones_like(x, dtype=F)
    for _ in range(n):
        r = (r * x).astype(F)
    return r


def _w_kind(kind, r, h):
    """kernel/poly6_kernel.rs:12-24, spiky_kernel.rs:12-24, viscosity_kernel.rs:12-32 (dim3); kind 0 = cubic spline"""
    if kind == 0:
        return _w(r, h)
    inside = r <= h
    if kind == 1:
        norm = F(315.0 / 64.0) / (F(np.pi) * _powi(h, 9))
        return np.where(inside, norm * _powi(h * h - r * r, 3), F(0)).astype(F)
    if kind == 2:
        norm = F(15.0) / (F(np.pi) * _powi(h, 6))
        return np.where(inside, norm * _powi(h - r, 3), F(0)).astype(F)
    norm = F(15.0) / (F(2.0) * F(np.pi) * _powi(h, 3))
    rs = np.where(r > 0, r, F(1))
    rr_hh = rs * rs / (h * h)
    val = norm * (rr_hh * (F(1.0) - rs / (F(2.0) * h)) + h / (F(2.0) * rs) - F(1.0))
    return np.where(inside & (r > 0), val, F(0)).astype(F)


def _dw_kind(kind, r, h):
    """poly6_kernel.rs:26-39, spiky_kernel.rs:26-39, viscosity_kernel.rs:34-50"""
    if kind == 0:
        return _dw(r, h)
    inside = r <= h
    if kind == 1:
        norm = F(315.0 / 64.0) / (F(np.pi) * _powi(h, 9))
        return np.where(inside, norm * _powi(h * h - r * r, 2) * r * F(-6.0), F(0)).astype(F)
    if kind == 2:
        norm = F(15.0) / (F(np.pi) * _powi(h, 6))
        return np.where(inside, -norm * _powi(h - r, 2) * F(3.0), F(0)).astype(F)
    norm = F(15.0) / (F(2.0) * F(np.pi) * _powi(h, 3))
    rs = np.where(r > 0, r, F(1))
    rr, hh = rs * rs, h * h
    val = norm * (F(-3.0) * rr / (F(2.0) * hh * h) + F(2.0) * rs / hh - h / (F(2.0) * rr))
    return np.where(inside & (r > 0), val, F(0)).astype(F)


class NumpyDFSPH:
    """Single-threaded dense restatement; fluids are concatenated, boundaries are concatenated."""

    def __init__(self, particle_radius, smoothing_factor=2.0, min_neighbors=20, kernel_density=0, kernel_gradient=0):
        self.kernel_density, self.kernel_gradient = kernel_density, kernel_gradient
        self.r = F(particle_radius)
        self.h = F(particle_radius) * F(smoothing_factor) * F(2.0)
        self.dt = F(0.0)
        self.inv_dt = F(0.0)
        self.fl = []  # dicts
        self.bd = []
        self.min_neighbors = min_neighbors
        self.max_div_iter, self.min_div_iter, self.max_div_err = 50, 1, F(0.1)
        self.max_p_iter, self.min_p_iter, self.max_dens_err = 50, 1, F(0.05)
        self.force_div = self.force_press = -1
        self.vc = None

    def add_fluid(self, positions, density0=1000.0, velocities=None, volumes=None, memberships=1, filter=0xFFFFFFFF):
        p = np.asarray(positions, F).reshape(-1, 3).copy()
        n = len(p)
        v = np.zeros((n, 3), F) if velocities is None else np.asarray(velocities, F).reshape(-1, 3).copy()
        vol = np.full(n, self.r * self.r * self.r * F(8.0 * 0.8), F) if volumes is None else np.asarray(volumes, F)
        self.fl.append(dict(p=p, v=v, vol=vol, rho0=F(density0), m=memberships, f=filter, forces=[]))
        return len(self.fl) - 1

    def push_force(self, fluid, kind, params):
        self.fl[fluid]["forces"].append((kind, [F(x) for x in params]))

    def add_boundary(self, positions, velocities=None, memberships=1, filter=0xFFFFFFFF, want_forces=False):
        p = np.asarray(positions, F).reshape(-1, 3).copy()
        v = np.zeros((len(p), 3), F) if velocities is None else np.asarray(velocities, F).reshape(-1, 3).copy()
        self.bd.append(dict(p=p, v=v, m=memberships, f=filter))
        return len(self.bd) - 1

    @staticmethod
    def _test(m1, f1, m2, f2):
        return (m1 & f2) != 0 and (m2 & f1) != 0

    def _gather(self):
        self.P = np.concatenate([f["p"] for f in self.fl])
        self.V = np.concatenate([f["v"] for f in self.fl])
        self.fid = np.concatenate([np.full(len(f["p"]), k) for k, f in enumerate(self.fl)])
        self.rho0 = np.concatenate([np.full(len(f["p"]), f["rho0"], F) for f in self.fl])
        self.mass = np.concatenate([f["vol"] * f["rho0"] for f in self.fl]).astype(F)
        self.vol = np.concatenate([f["vol"] for f in self.fl]).astype(F)
        if self.vc is None or len(self.vc) != len(self.P):
            self.vc = np.zeros_like(self.P)
        if self.bd:
            self.BP = np.concatenate([b["p"] for b in self.bd])
            self.BV = np.concatenate([b["v"] for b in self.bd])
            self.bid = np.concatenate([np.full(len(b["p"]), k) for k, b in enumerate(self.bd)])
        else:
            self.BP = np.zeros((0, 3), F)
            self.BV = np.zeros((0, 3), F)
            self.bid = np.zeros(0, int)

    def _pairs(self, A, B):
        d = (A[:, None, :] - B[None, :, :]).astype(F)
        d2 = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F)
        return d, d2

    def _kernels(self, d, d2, mask):
        r = np.sqrt(d2).astype(F)
        W = np.where(mask, _w_kind(self.kernel_density, r, self.h), F(0)).astype(F)
        ok = d2 > EPS * EPS
        rs = np.where(ok, r, F(1))
        dirs = (d / rs[..., None]).astype(F)
        G = np.where((mask & ok)[..., None], dirs * _dw_kind(self.kernel_gradient, r, self.h)[..., None], F(0)).astype(F)
        return W, G

    def contacts(self):
        self._gather()
        h2 = self.h * self.h
        nf, nb = len(self.fl), len(self.bd)
        gf = np.array([[a == b or self._test(self.fl[a]["m"], self.fl[a]["f"], self.fl[b]["m"], self.fl[b]["f"])
                        for b in range(nf)] for a in range(nf)], bool).reshape(nf, nf)
        d, d2 = self._pairs(self.P, self.P)
        self.Mff = (d2 <= h2) & gf[self.fid[:, None], self.fid[None, :]]
        self.same = self.fid[:, None] == self.fid[None, :]
        self.Wff, self.Gff = self._kernels(d, d2, self.Mff)
        self.Dff, self.D2ff = d, d2
        if nb:
            gfb = np.array([[self._test(self.fl[a]["m"], self.fl[a]["f"], self.bd[b]["m"], self.bd[b]["f"])
                             for b in range(nb)] for a in range(nf)], bool).reshape(nf, nb)
            d, d2 = self._pairs(self.P, self.BP)
            self.Mfb = (d2 <= h2) & gfb[self.fid[:, None], self.bid[None, :]]
            self.Wfb, self.Gfb = self._kernels(d, d2, self.Mfb)
            self.Dfb, self.D2fb = d, d2
            gbb = np.array([[a == b or self._test(self.bd[a]["m"], self.bd[a]["f"], self.bd[b]["m"], self.bd[b]["f"])
                             for b in range(nb)] for a in range(nb)], bool).reshape(nb, nb)
            d, d2 = self._pairs(self.BP, self.BP)
            Mbb = (d2 <= h2) & gbb[self.bid[:, None], self.bid[None, :]]
            Wbb, _ = self._kernels(d, d2, Mbb)
            self.bvol = (F(1.0) / Wbb.sum(axis=1, dtype=F)).astype(F)
        else:
            n = len(self.P)
            self.Mfb = np.zeros((n, 0), bool)
            self.Wfb = np.zeros((n, 0), F)
            self.Gfb = np.zeros((n, 0, 3), F)
            self.Dfb = np.zeros((n, 0, 3), F)
            self.D2fb = np.zeros((n, 0), F)
            self.bvol = np.zeros(0, F)
        self.nff = self.Mff.sum(axis=1)
        self.nfb = self.Mfb.sum(axis=1)
        # boundary pseudo mass seen by fluid i: vol_b * rho0_i
        self.mb = (self.bvol[None, :] * self.rho0[:, None]).astype(F)

    def densities_alphas(self):
        self.dens = ((self.mass[None, :] * self.Wff).sum(axis=1, dtype=F) + (self.mb * self.Wfb).sum(axis=1, dtype=F)).astype(F)
        gf = (self.Gff * self.mass[None, :, None]).astype(F)
        gb = (self.Gfb * self.mb[..., None]).astype(F)
        sq = (gf * gf).sum(axis=(1, 2), dtype=F) + (gb * gb).sum(axis=(1, 2), dtype=F)
        gs = gf.sum(axis=1, dtype=F) + gb.sum(axis=1, dtype=F)
        den = (sq + (gs * gs).sum(axis=1, dtype=F)).astype(F)
        self.alpha = np.where(den <= F(1.0e-5), F(0), F(1.0) / np.where(den == 0, F(1), den)).astype(F)

    def _mean_max(self, per_particle):
        err = F(0)
        for k in range(len(self.fl)):
            sel = self.fid == k
            if sel.any():
                err = max(err, F(per_particle[sel].sum(dtype=F) / F(sel.sum())))
        return err

    def divergences(self):
        vs = (self.V + self.vc).astype(F)
        dv = (vs[:, None, :] - vs[None, :, :]).astype(F)
        d = ((dv * self.Gff).sum(axis=2, dtype=F) * self.mass[None, :]).sum(axis=1, dtype=F)
        d = d + (((vs[:, None, :] * self.Gfb).sum(axis=2, dtype=F)) * self.mb).sum(axis=1, dtype=F)
        d = np.maximum(d, F(0)).astype(F)
        d = np.where(self.nff + self.nfb < self.min_neighbors, F(0), d).astype(F)
        self.div = d
        return self._mean_max(d / self.rho0)

    def vc_divergence(self):
        k = (self.div * self.alpha).astype(F)
        coeff = (-(k[:, None] + k[None, :]) * self.mass[None, :]).astype(F)
        self.vc = (self.vc + (self.Gff * coeff[..., None]).sum(axis=1, dtype=F)).astype(F)
        cb = (-k[:, None] * self.mb).astype(F)
        self.vc = (self.vc + (self.Gfb * cb[..., None]).sum(axis=1, dtype=F)).astype(F)

    def predicted(self):
        vs = (self.V + self.vc).astype(F)
        dv = (vs[:, None, :] - vs[None, :, :]).astype(F)
        delta = ((dv * self.Gff).sum(axis=2, dtype=F) * self.mass[None, :]).sum(axis=1, dtype=F)
        dvb = (vs[:, None, :] - self.BV[None, :, :]).astype(F)
        delta = delta + ((dvb * self.Gfb).sum(axis=2, dtype=F) * self.mb).sum(axis=1, dtype=F)
        self.pred = (self.dens + delta * self.dt).astype(F)
        e = np.where(self.pred < self.rho0, F(0), self.pred / self.rho0 - F(1)).astype(F)
        return self._mean_max(e)

    def vc_pressure(self):
        k = ((self.pred - self.rho0) * self.alpha).astype(F)
        kp = np.maximum(k, F(0))
        kij = (kp[:, None] + kp[None, :]).astype(F)
        coeff = np.where(kij > 0, kij * self.mass[None, :] * self.inv_dt, F(0)).astype(F)
        self.vc = (self.vc - (self.Gff * coeff[..., None]).sum(axis=1, dtype=F)).astype(F)
        cb = (kp[:, None] * self.mb * self.inv_dt).astype(F)
        self.vc = (self.vc - (self.Gfb * cb[..., None]).sum(axis=1, dtype=F)).astype(F)

    def _forces(self, g):
        acc = np.tile(np.asarray(g, F), (len(self.P), 1))
        h = self.h
        for fi, fl in enumerate(self.fl):
            sel = self.fid == fi
            sm = self.Mff & self.same & sel[:, None]
            for force_index, (kind, p) in enumerate(fl["forces"]):
                if kind == 3:  # Becker 2009 (becker2009_elasticity.rs:84-334); rotations by SVD polar decomposition
                    acc = self._becker(acc, fi, force_index, p, sel)
                elif kind == 0:  # XSPH
                    cf, cb = p[0], p[1]
                    dv = (self.V[None, :, :] - self.V[:, None, :]).astype(F)
                    c = np.where(sm, cf * self.Wff * self.vol[None, :] * self.rho0[:, None] / self.dens[None, :], F(0)).astype(F)
                    a = (dv * c[..., None]).sum(axis=1, dtype=F)
                    if cb != 0 and len(self.BP):
                        dvb = (self.BV[None, :, :] - self.V[:, None, :]).astype(F)
                        c2 = np.where(self.Mfb & sel[:, None], cb * self.Wfb * self.mb / self.dens[:, None], F(0)).astype(F)
                        a = a + (dvb * c2[..., None]).sum(axis=1, dtype=F)
                    acc = (acc + a * self.inv_dt).astype(F)
                elif kind == 1:  # artificial viscosity
                    cf, cb, al, be, cs = p[0], p[1], p[2], p[3], p[4]
                    vij = (self.V[:, None, :] - self.V[None, :, :]).astype(F)
                    vr = (self.Dff * vij).sum(axis=2, dtype=F)
                    mu = (h * vr / (self.D2ff + h * h * F(0.01))).astype(F)
                    davg = ((self.dens[:, None] + self.dens[None, :]) * F(0.5)).astype(F)
                    c = np.where(sm & (vr < 0), cf * (cs * al * mu - be * mu * mu) * (self.mass[None, :] / davg), F(0)).astype(F)
                    acc = (acc + (self.Gff * c[..., None]).sum(axis=1, dtype=F)).astype(F)
                    if cb != 0 and len(self.BP):
                        vib = (self.V[:, None, :] - self.BV[None, :, :]).astype(F)
                        vr = (self.Dfb * vib).sum(axis=2, dtype=F)
                        mu = (h * vr / (self.D2fb + h * h * F(0.01))).astype(F)
                        c = np.where(self.Mfb & sel[:, None] & (vr < 0),
                                     cb * (cs * al * mu - be * mu * mu) * (self.mb / self.dens[:, None]), F(0)).astype(F)
                        acc = (acc + (self.Gfb * c[..., None]).sum(axis=1, dtype=F)).astype(F)
                elif kind == 2:  # Akinci 2013
                    gamma, adh = p[0], p[1]
                    c = np.where(sm, self.mass[None, :] / self.dens[None, :], F(0)).astype(F)
                    nrm = ((self.Gff * c[..., None]).sum(axis=1, dtype=F) * h).astype(F)
                    r = np.sqrt(self.D2ff).astype(F)
                    ok = self.D2ff > EPS * EPS
                    dirs = self.Dff / np.where(ok, r, F(1))[..., None]
                    norm_c = F(32.0) / (F(np.pi) * h ** 9)
                    hr3 = ((h - r) ** 3 * r ** 3).astype(F)
                    coh = norm_c * np.where(r <= h / F(2), F(2) * hr3 - h ** 6 / F(64), np.where(r <= h, hr3, F(0)))
                    cohv = np.where(ok[..., None], dirs * coh[..., None], F(0)).astype(F)
                    coh_acc = cohv * (-gamma * self.mass[None, :, None])
                    curv = (nrm[:, None, :] - nrm[None, :, :]) * (-gamma)
                    kij = (F(2) * self.rho0[:, None] / (self.dens[:, None] + self.dens[None, :])).astype(F)
                    tot = np.where(sm[..., None], (curv + coh_acc) * kij[..., None], F(0)).astype(F)
                    acc = (acc + tot.sum(axis=1, dtype=F)).astype(F)
                    if adh != 0 and len(self.BP):
                        r = np.sqrt(self.D2fb).astype(F)
                        ok = self.D2fb > EPS * EPS
                        dirs = self.Dfb / np.where(ok, r, F(1))[..., None]
                        inr = (r > h / F(2)) & (r <= h)
                        ak = np.where(inr, F(0.007) / h ** F(3.25) *
                                      np.maximum(-F(4) * r * r / h + F(6) * r - F(2) * h, F(0)) ** F(0.25), F(0)).astype(F)
                        av = np.where((ok & self.Mfb & sel[:, None])[..., None], dirs * ak[..., None], F(0)).astype(F)
                        acc = (acc - (av * (adh * self.mb)[..., None]).sum(axis=1, dtype=F)).astype(F)
                elif kind == 4:  # He 2014 (he2014_surface_tension.rs:40-178)
                    cf, cb = F(p[0]), F(p[1])
                    mfb = self.Mfb & sel[:, None]
                    colors = (np.where(sm, self.Wff * self.mass[None, :] / self.dens[None, :], F(0)).sum(axis=1, dtype=F)
                              + np.where(mfb, self.Wfb * self.bvol[None, :], F(0)).sum(axis=1, dtype=F)).astype(F)
                    cj = np.where(sm, colors[None, :] * self.mass[None, :] / self.dens[None, :], F(0)).astype(F)
                    gradc = (self.Gff * cj[..., None]).sum(axis=1, dtype=F)
                    q = (gradc / np.where(sel, colors, F(1))[:, None]).astype(F)
                    gc = np.where(sel, (q * q).sum(axis=1, dtype=F), F(0)).astype(F)
                    mi = self.mass
                    if cf != 0:
                        c = np.where(sm, mi[:, None] / self.dens[:, None] * self.mass[None, :] / self.dens[None, :]
                                     * (gc[:, None] + gc[None, :]) / F(2), F(0)).astype(F)
                        a = (self.Gff * c[..., None]).sum(axis=1, dtype=F) * (cf / (F(2) * mi))[:, None]
                        acc = (acc + np.where(sel[:, None], a, F(0))).astype(F)
                    if cb != 0 and len(self.BP):
                        c = np.where(mfb, mi[:, None] / self.dens[:, None] * self.mb / self.rho0[:, None] * gc[:, None] * cb * F(0.25),
                                     F(0)).astype(F)
                        a = (self.Gfb * c[..., None]).sum(axis=1, dtype=F) / mi[:, None]
                        acc = (acc + np.where(sel[:, None], a, F(0))).astype(F)
                elif kind == 5:  # WCSPH fluid term (wcsph_surface_tension.rs:45-63)
                    cf = F(p[0])
                    c = np.where(sm, -cf * self.Wff * self.mass[None, :] / self.mass[:, None], F(0)).astype(F)
                    acc = (acc + (self.Dff * c[..., None]).sum(axis=1, dtype=F)).astype(F)
                elif kind == 6:  # DFSPHViscosity (dfsph_viscosity.rs:133-324), dense restatement with LAPACK inverses
                    visc, min_it, max_it, max_err = F(p[0]), int(p[1]), int(p[2]), F(p[3])
                    idx = np.nonzero(sel)[0]
                    G = self.Gff
                    Z = np.zeros_like(G[..., 0])
                    mat = np.stack([np.stack([G[..., 0] * 2, Z, Z], -1), np.stack([Z, G[..., 1] * 2, Z], -1),
                                    np.stack([Z, Z, G[..., 2] * 2], -1), np.stack([G[..., 1], G[..., 0], Z], -1),
                                    np.stack([G[..., 2], Z, G[..., 0]], -1), np.stack([Z, G[..., 2], G[..., 1]], -1)], -2).astype(F)  # N,N,6,3
                    sc = np.where(sm, self.mass[None, :] / (F(2) * self.dens[:, None]), F(0)).astype(F)
                    gi = (mat * sc[..., None, None]).astype(F)
                    sq = (np.einsum("ijrk,ijck->ijrc", gi, gi).astype(F) / self.dens[:, None, None, None]).sum(axis=1, dtype=F)
                    gs = gi.sum(axis=1, dtype=F)
                    den = (sq + np.einsum("irk,ick->irc", gs, gs).astype(F) / self.dens[:, None, None]).astype(F)
                    betas = np.zeros((len(self.P), 6, 6), F)
                    for i in idx:
                        d = den[i].copy()
                        dg = np.diag(d).copy()
                        inv_diag = np.where(np.abs(dg) < F(1e-6), F(1), F(1) / np.where(dg == 0, F(1), dg)).astype(F)
                        d[:, :3] *= inv_diag[:, None]
                        if abs(np.linalg.det(d.astype(np.float64))) >= 1e-6:
                            b = np.linalg.inv(d.astype(np.float64)).astype(F)
                            b[:, :3] *= inv_diag[None, :3]
                            betas[i] = b
                    dtl = self.dt

                    def rates(a):
                        vv = (self.V + a * dtl).astype(F)
                        vji = (vv[None, :, :] - vv[:, None, :]).astype(F)
                        r6 = np.stack([F(2) * vji[..., 0] * G[..., 0], F(2) * vji[..., 1] * G[..., 1], F(2) * vji[..., 2] * G[..., 2],
                                       vji[..., 0] * G[..., 1] + vji[..., 1] * G[..., 0], vji[..., 0] * G[..., 2] + vji[..., 2] * G[..., 0],
                                       vji[..., 1] * G[..., 2] + vji[..., 2] * G[..., 1]], -1).astype(F)
                        return (r6 * sc[..., None]).sum(axis=1, dtype=F)

                    target = (rates(acc) * (F(1) - visc)).astype(F)
                    self.visc_iters = 0
                    for it in range(max_it):
                        err6 = (rates(acc) - target).astype(F)
                        avg = F(np.abs(err6[idx]).sum(axis=1, dtype=F).sum(dtype=F) / F(6) / F(max(len(idx), 1)))
                        self.visc_err = avg
                        if avg <= max_err and it >= min_it:
                            break
                        u = (np.einsum("irk,ik->ir", betas, err6).astype(F) / (self.dens * self.dens)[:, None]).astype(F)
                        co = np.where(sm[..., None], (u[:, None, :] + u[None, :, :]) * (self.mass[None, :, None] / F(2)), F(0)).astype(F)
                        t = np.einsum("ijrk,ijr->ijk", mat, co).astype(F)
                        a = t.sum(axis=1, dtype=F) * (self.mass * self.inv_dt)[:, None]
                        acc = (acc + np.where(sel[:, None], a, F(0))).astype(F)
                        self.visc_iters += 1
                else:
                    raise NotImplementedError(kind)
        return acc

    def _becker(self, acc, fi, force_index, p, sel):
        """Dense restatement of Becker2009Elasticity::solve.  The reference extracts the rotation of A_pq with nalgebra's
        iterative `from_matrix_eps` (warm-started, <= 20 iterations); here it is the orthogonal polar factor from an f64
        SVD — a different algorithm that agrees with the converged iteration, so it independently checks the oracle's
        restatement of that third-party routine."""
        h = self.h
        young, poisson, nonlinear = F(p[0]), F(p[1]), p[2] != 0
        one, two = F(1), F(2)
        d0 = (young * (one - poisson)) / ((one + poisson) * (one - two * poisson))     # elasticity_coefficients :15-26
        d1 = (young * poisson) / ((one + poisson) * (one - two * poisson))
        d2 = (young * (one - two * poisson)) / (two * (one + poisson) * (one - two * poisson))
        idx = np.nonzero(sel)[0]
        n = len(idx)
        P = self.P[idx]
        mass = self.mass[idx]
        st = self.__dict__.setdefault("_becker_state", {}).get((fi, force_index))
        if st is None or len(st["pos0"]) != n:                                           # init :84-113
            old = st["vol0"] if st is not None else np.zeros(0, F)
            d = (P[:, None, :] - P[None, :, :]).astype(F)
            dd = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F)
            M0 = dd <= h * h                                                             # compute_self_contacts, self included
            W0, G0 = self._kernels(d, dd, M0)
            raw = np.zeros(n, F)
            raw[:min(n, len(old))] = old[:min(n, len(old))]                              # Vec::resize keeps old entries (:89)
            raw = (raw + two * (W0 * mass[None, :]).sum(axis=1, dtype=F)).astype(F)      # both ends of every ordered pair
            st = dict(pos0=P.copy(), M0=M0, W0=W0, G0=G0, vol0=(mass / raw).astype(F))
            self._becker_state[(fi, force_index)] = st
        M0, W0, G0, vol0, P0 = st["M0"], st["W0"], st["G0"], st["vol0"], st["pos0"]
        p_ji = (P[None, :, :] - P[:, None, :]).astype(F)                                 # [i, j] = p_j - p_i
        p0_ji = (P0[None, :, :] - P0[:, None, :]).astype(F)
        coeff = np.where(M0, W0 * mass[None, :], F(0)).astype(F)
        a_pq = np.einsum("ijr,ijc->irc", p_ji, p0_ji * coeff[..., None]).astype(F)      # compute_rotations :115-137
        R = np.zeros((n, 3, 3), F)
        for i in range(n):
            u, _, vt = np.linalg.svd(a_pq[i].astype(np.float64))
            r = u @ vt
            if np.linalg.det(r) < 0:
                u[:, -1] *= -1
                r = u @ vt
            R[i] = r.astype(F)
        rt_p = np.einsum("icr,ijc->ijr", R, p_ji).astype(F)                              # R_i^T p_ji  (inverse_transform_vector)
        u_ji = (rt_p - p0_ji).astype(F)
        gv = np.where(M0[..., None], G0 * vol0[None, :, None], F(0)).astype(F)           # gradient * volumes0[j]
        grad_tr = np.einsum("ijr,ijc->irc", gv, u_ji).astype(F)                          # compute_stresses :139-262
        k = F(0.564)
        if nonlinear:
            J = (grad_tr + np.eye(3, dtype=F)[None]).astype(F)
            JJt = np.einsum("irk,ick->irc", J, J).astype(F)
            e = np.stack([JJt[:, 0, 0] - one, JJt[:, 1, 1] - one, JJt[:, 2, 2] - one], -1).astype(F)
            sh = np.stack([JJt[:, 1, 0], JJt[:, 2, 0], JJt[:, 2, 1]], -1).astype(F)
            s012 = np.stack([d0 * e[:, 0] + d1 * e[:, 1] + d1 * e[:, 2], d1 * e[:, 0] + d0 * e[:, 1] + d1 * e[:, 2],
                             d1 * e[:, 0] + d1 * e[:, 1] + d0 * e[:, 2]], -1).astype(F) * k
        else:
            e = np.stack([grad_tr[:, 0, 0], grad_tr[:, 1, 1], grad_tr[:, 2, 2]], -1).astype(F)
            sh = np.stack([grad_tr[:, 1, 0] + grad_tr[:, 0, 1], grad_tr[:, 2, 0] + grad_tr[:, 0, 2],
                           grad_tr[:, 1, 2] + grad_tr[:, 2, 1]], -1).astype(F)
            s012 = np.stack([d0 * e[:, 0] + d1 * e[:, 1] + d1 * e[:, 2], d1 * e[:, 0] + d0 * e[:, 1] + d1 * e[:, 2],
                             d1 * e[:, 0] + d1 * e[:, 1] + d0 * e[:, 2]], -1).astype(F)
        s345 = (sh * k * d2).astype(F)
        S = np.zeros((n, 3, 3), F)                                                       # sym_mat_mul_vec layout :28-39
        S[:, 0, 0], S[:, 1, 1], S[:, 2, 2] = s012[:, 0], s012[:, 1], s012[:, 2]
        S[:, 0, 1] = S[:, 1, 0] = s345[:, 0]
        S[:, 0, 2] = S[:, 2, 0] = s345[:, 1]
        S[:, 1, 2] = S[:, 2, 1] = s345[:, 2]
        d_ij = gv                                                                        # gradient * volumes0[j]
        d_ji = np.where(M0[..., None], G0 * (-vol0)[:, None, None], F(0)).astype(F)      # gradient * (-volumes0[i])
        sd_ij = np.einsum("irc,ijc->ijr", S, d_ij).astype(F)                             # stress[i] * d_ij
        sd_ji = np.einsum("jrc,ijc->ijr", S, d_ji).astype(F)                             # stress[j] * d_ji
        if nonlinear:
            f_ji = ((sd_ij + np.einsum("irc,ijc->ijr", grad_tr, sd_ij)) * (-vol0)[:, None, None]).astype(F)
            f_ij = ((sd_ji + np.einsum("jrc,ijc->ijr", grad_tr, sd_ji)) * (-vol0)[None, :, None]).astype(F)
        else:
            f_ji = (sd_ij * (-vol0)[:, None, None]).astype(F)
            f_ij = (sd_ji * (-vol0)[None, :, None]).astype(F)
        force = ((np.einsum("jrc,ijc->ijr", R, f_ij) - np.einsum("irc,ijc->ijr", R, f_ji)) * F(0.5)).astype(F)
        force = np.where(M0[..., None], force, F(0))
        a = (force.sum(axis=1, dtype=F) / mass[:, None]).astype(F)
        out = acc.copy()
        out[idx] = (out[idx] + a).astype(F)
        return out

    def step(self, dt, gravity=(0.0, -9.81, 0.0)):
        """liquid_world.rs:67-158 + dfsph_solver.rs:667-708"""
        self.contacts()
        self.densities_alphas()
        self.n_div_iter = 0
        nmax = self.force_div + 1 if self.force_div >= 0 else self.max_div_iter
        for i in range(nmax):
            err = self.divergences()
            if self.force_div >= 0:
                if i >= self.force_div:
                    break
            elif err <= self.max_div_err * self.inv_dt * F(0.01) and i >= self.min_div_iter:
                break
            self.vc_divergence()
            self.n_div_iter += 1
        self.V = (self.V + self.vc).astype(F)
        self.vc = np.zeros_like(self.vc)
        acc = self._forces(gravity)
        self.acc = acc
        self.dt = F(dt)
        self.inv_dt = F(0) if self.dt == 0 else F(1.0) / self.dt
        self.vc = (self.vc + acc * self.dt).astype(F)
        self.n_press_iter = 0
        nmax = self.force_press + 1 if self.force_press >= 0 else self.max_p_iter
        for i in range(nmax):
            err = self.predicted()
            if self.force_press >= 0:
                if i >= self.force_press:
                    break
            elif err <= self.max_dens_err and i >= self.min_p_iter:
                break
            self.vc_pressure()
            self.n_press_iter += 1
        self.P = (self.P + (self.V + self.vc) * self.dt).astype(F)
        o = 0
        for f in self.fl:
            n = len(f["p"])
            f["p"] = self.P[o:o + n].copy()
            f["v"] = self.V[o:o + n].copy()
            o += n

    def step_iisph(self, dt, gravity=(0.0, -9.81, 0.0), omega=F(0.5)):
        """liquid_world.rs:67-158 + iisph_solver.rs:643-711 (dense restatement).  Keeps dii, aii and the last iteration's
        dij_pjl (dijpj) as attributes."""
        self.contacts()
        self.densities_alphas()
        if not hasattr(self, "press") or len(self.press) != len(self.P):
            self.press = np.zeros(len(self.P), F)
        acc = self._forces(gravity)            # predict_advection sees the previous dt / inv_dt
        self.acc = acc
        self.dt = F(dt)
        self.inv_dt = F(0) if self.dt == 0 else F(1.0) / self.dt
        dt = self.dt
        self.vc = (self.vc + acc * dt).astype(F)
        rho = self.dens
        factor = (-dt * dt / (rho * rho)).astype(F)
        dii = ((self.Gff * (self.mass[None, :] * factor[:, None])[..., None]).sum(axis=1, dtype=F) +
               (self.Gfb * (self.mb * factor[:, None])[..., None]).sum(axis=1, dtype=F)).astype(F)
        self.press = (self.press * F(0.5)).astype(F)
        self.predicted()
        fac2 = (dt * dt * self.mass / (rho * rho)).astype(F)
        dji = (self.Gff * fac2[:, None, None]).astype(F)
        aii = ((((dii[:, None, :] - dji) * self.Gff).sum(axis=2, dtype=F) * self.mass[None, :]).sum(axis=1, dtype=F))
        djib = (self.Gfb * fac2[:, None, None]).astype(F)
        aii = (aii + (((dii[:, None, :] - djib) * self.Gfb).sum(axis=2, dtype=F) * self.mb).sum(axis=1, dtype=F)).astype(F)
        self.dii, self.aii = dii, aii
        self.n_press_iter = 0
        nmax = self.force_press if self.force_press >= 0 else self.max_p_iter
        for i in range(nmax):
            p = self.press
            dijpj = ((self.Gff * (-self.mass * p / (rho * rho))[None, :, None]).sum(axis=1, dtype=F) * (dt * dt)).astype(F)
            self.dijpj = dijpj   # the last iteration's, as the solver keeps it
            fct = (dijpj[:, None, :] - dii[None, :, :] * p[None, :, None] - (dijpj[None, :, :] - dji * p[:, None, None])).astype(F)
            ssum = ((fct * self.Gff).sum(axis=2, dtype=F) * self.mass[None, :]).sum(axis=1, dtype=F)
            ssum = (ssum + ((dijpj[:, None, :] * self.Gfb).sum(axis=2, dtype=F) * self.mb).sum(axis=1, dtype=F)).astype(F)
            ok = np.abs(aii) > F(1.0e-9)
            safe = np.where(ok, aii, F(1))
            npr = ((F(1) - omega) * p + omega * (self.rho0 - self.pred - ssum) / safe).astype(F)
            pos = ok & (npr > 0)
            err = np.where(pos, (-ssum - aii * npr) / self.rho0, F(0)).astype(F)
            self.press = np.where(pos, npr, F(0)).astype(F)
            self.n_press_iter += 1
            if self.force_press < 0 and self._mean_max(err) <= self.max_dens_err and i >= self.min_p_iter:
                break
        p = self.press
        pr = (p / (rho * rho)).astype(F)
        c = (dt * self.mass[None, :] * (pr[:, None] + pr[None, :])).astype(F)
        self.vc = (self.vc - (self.Gff * c[..., None]).sum(axis=1, dtype=F)).astype(F)
        cb = (self.mb * pr[:, None] * dt).astype(F)
        self.vc = (self.vc - (self.Gfb * cb[..., None]).sum(axis=1, dtype=F)).astype(F)
        self.V = (self.V + self.vc).astype(F)
        self.P = (self.P + self.V * dt).astype(F)
        self.vc = np.zeros_like(self.vc)
        o = 0
        for f in self.fl:
            n = len(f["p"])
            f["p"] = self.P[o:o + n].copy()
            f["v"] = self.V[o:o + n].copy()
            o += n

    def read_fluid(self, k):
        return self.fl[k]["p"].copy(), self.fl[k]["v"].copy()
