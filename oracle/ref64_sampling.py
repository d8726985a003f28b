"""Float64 reference of salva3d's ray sampling (sampling/ray_sampling.rs:27-231, 3-D branch) for checking
sph_world_sample_shape.  Test infrastructure only.

The traversal is restated exactly in float32 (numpy): the AABB, its loosening, `origin`, the running sums that place the
rays, the one-step-in first row of the y and z ray families, and every operation after a crossing is known (toi, impact,
quotient, ceil / floor / round, the sub / 10 advance).  Only the crossing coordinate X itself is not restated bit for bit:
it is computed in float64 from the float32 inputs, with a bound eX on how far the device's float32 evaluation may lie
from it.  Every later operation is a monotone function of X, so the reference evaluates it at both ends of
[X - eX, X + eX]: a decision is undecided exactly when the two ends disagree.  Undecided quantisations mark their keys
undecided; an undecided advance (a crossing within its bound of o + sub / 10), a grazing ray (a ball or capsule tangent)
or a heightfield ray at a vertex height of its profile makes the rest of that ray undecided: every key on the ray's line
from that point on.  Cuboid crossings are exact float32 values (eX = 0), so cuboids are decided throughout.

Heightfields follow the project's contract (DESIGN.md section 11): rows of the height matrix along z, columns along x,
the field centred on [-0.5, 0.5] * scale in x and z, heights times scale[1], and cell (i, j) split along its
(x0, z1)-(x1, z0) diagonal.  The diagonal and the row / column orientation are parameters (`bugs`), so that a sampler
with either one swapped is caught, as are the other plausible sampler bugs listed in BUGS.
"""
import math

import numpy as np

F32 = np.float32
U = 2.0 ** -24  # unit roundoff of float32
BALL, CUBOID, CAPSULE, HEIGHTFIELD = 1, 2, 3, 4
KEY_BITS = 21
KEY_LIM = 1 << KEY_BITS

# plausible sampler bugs the reference can be run with (each one a set member of `bugs`)
BUGS = ("ceil_floor_swapped",   # floor for entries, ceil for exits
        "floor_across",         # floor instead of round across the ray axis
        "no_loosen",            # the AABB is not loosened by sub
        "no_half_offset",       # origin = loosened mins, without + sub / 2
        "times_sub",            # ray coordinates origin + n * sub instead of running sums
        "no_skip",              # no sub / 10 advance: every crossing after the impact counts
        "skip_keeps_parity",    # crossings passed over by the advance still toggle entry / exit
        "exclusive_end",        # sample_segment's range excludes its end
        "hf_zigzag",            # heightfield cells split along the (x0, z0)-(x1, z1) diagonal
        "hf_rows_along_x",      # heightfield rows along x and columns along z
        "fma_unquantize")       # unquantise with one rounding (a fused multiply-add)


def _f(x):
    return F32(x)


def _down(x):
    """Largest float32 <= x (x a Python float)."""
    f = F32(x)
    return f if float(f) <= x else np.nextafter(f, F32(-np.inf))


def _up(x):
    f = F32(x)
    return f if float(f) >= x else np.nextafter(f, F32(np.inf))


def key(c):
    return (int(c[0]) << (2 * KEY_BITS)) | (int(c[1]) << KEY_BITS) | int(c[2])


def unkey(k):
    k = np.asarray(k, np.int64)
    return np.stack([(k >> (2 * KEY_BITS)) & (KEY_LIM - 1), (k >> KEY_BITS) & (KEY_LIM - 1), k & (KEY_LIM - 1)], axis=1)


class Shape:
    """kind BALL (radius), CUBOID (half extents), CAPSULE (half height, radius) or HEIGHTFIELD (heights (nrows, ncols), scale)."""

    def __init__(self, kind, params=(), heights=None, scale=None):
        self.kind = kind
        self.params = [F32(p) for p in params]
        self.heights = None if heights is None else np.asarray(heights, F32)
        self.scale = None if scale is None else np.asarray(scale, F32)


def aabb(shape):
    """shape.compute_aabb(&Isometry::identity()) in float32."""
    z = F32(0)
    if shape.kind == BALL:
        r = shape.params[0]
        return np.array([z - r] * 3, F32), np.array([z + r] * 3, F32)
    if shape.kind == CUBOID:
        he = shape.params
        return np.array([z - h for h in he], F32), np.array([z + h for h in he], F32)
    if shape.kind == CAPSULE:
        hh, r = shape.params
        return np.array([z - r, -hh - r, z - r], F32), np.array([z + r, hh + r, z + r], F32)
    H, s = shape.heights, shape.scale
    hx, hz = s[0] * F32(0.5), s[2] * F32(0.5)
    return np.array([-hx, H.min() * s[1], -hz], F32), np.array([hx, H.max() * s[1], hz], F32)


def grid(shape, particle_rad, bugs=()):
    """sub, sub / 10, origin and the three per-axis tables of ray coordinates (ray_sampling.rs:33-38, 55-72)."""
    sub = F32(particle_rad) * F32(2)
    mins, maxs = aabb(shape)
    if "no_loosen" not in bugs:
        mins, maxs = mins - sub, maxs + sub
    origin = mins if "no_half_offset" in bugs else mins + sub / F32(2)
    tabs = []
    for a in range(3):
        t = []
        c = origin[a]
        while c < maxs[a]:  # curr[k] += sub while curr[k] < maxs[k]
            t.append(c)
            c = F32(origin[a] + F32(len(t)) * sub) if "times_sub" in bugs else F32(c + sub)
        tabs.append(np.array(t, F32))
    return sub, sub / F32(10), origin.astype(F32), tabs


# -- crossings: exact X (float64 of float32 inputs) with the bound eX of the device's float32 evaluation ---------------------
def _sqrt_pair(S, eS, shift=0.0, eshift=0.0):
    """The two crossings +-(shift + sqrt(S)) of S with error eS; (crossings, undecided_from)."""
    if S < -eS:
        return [], math.inf
    if abs(S) <= eS:
        return [], -math.inf  # grazing: whether the ray hits is undecided
    T = shift + math.sqrt(S)
    eT = eS / math.sqrt(S) + eshift + 3 * U * T
    return [(-T, eT), (T, eT)], math.inf


class _HF:
    """The heightfield surface as the exact function of (x, z) the contract describes."""

    def __init__(self, shape, bugs):
        H = shape.heights.astype(np.float64)
        if "hf_rows_along_x" in bugs:
            H = H.T
        self.H = H  # H[row along z, column along x]
        self.nr, self.nc = H.shape
        s = shape.scale
        self.sx, self.sy, self.sz = float(s[0]), float(s[1]), float(s[2])
        self.hx, self.hz = float(s[0] * F32(0.5)), float(s[2] * F32(0.5))
        self.dx, self.dz = self.sx / (self.nc - 1), self.sz / (self.nr - 1)
        self.zig = "hf_zigzag" in bugs
        Hs = H * self.sy
        rng = float(Hs.max() - Hs.min())
        self.hmax = float(np.abs(Hs).max())
        ev = 8 * U * (self.nr + self.nc + 2)  # |fraction error| of the device's cell coordinate
        self.ev = ev
        self.ex = 6 * U * max(self.sx, self.sz)  # |grid position error|
        self.Ef = 2 * ev * rng + 10 * U * self.hmax  # |profile height error|, before the ray height's share

    def cell(self, c, half, d, cells):
        t = (c + half) / d
        i = min(max(int(math.floor(t)), 0), cells - 1)
        return i, t - i

    def flat_cell(self, x, z):
        """The common height of the cell under (x, z) when its four corners are equal and (x, z) is further than the device's
        cell-coordinate error from the cell's edges (the device then takes this cell and computes h + u * 0 + v * 0), else
        None."""
        if self.zig:
            return None
        j, u = self.cell(x, self.hx, self.dx, self.nc - 1)
        i, v = self.cell(z, self.hz, self.dz, self.nr - 1)
        c = self.H[i:i + 2, j:j + 2]
        if c.min() != c.max() or not (self.ev < u < 1 - self.ev and self.ev < v < 1 - self.ev):
            return None
        return c[0, 0]

    def height(self, x, z):
        j, u = self.cell(x, self.hx, self.dx, self.nc - 1)
        i, v = self.cell(z, self.hz, self.dz, self.nr - 1)
        H = self.H
        h00, h10, h01, h11 = H[i, j], H[i, j + 1], H[i + 1, j], H[i + 1, j + 1]  # h10: (x1, z0), h01: (x0, z1)
        if self.zig:
            if u >= v:
                h = h00 + u * (h10 - h00) + v * (h11 - h10)
            else:
                h = h00 + v * (h01 - h00) + u * (h11 - h01)
        elif u + v <= 1:
            h = h00 + u * (h10 - h00) + v * (h01 - h00)
        else:
            h = h11 + (1 - u) * (h01 - h11) + (1 - v) * (h10 - h11)
        return h * self.sy

    def profile(self, along, c):
        """Breakpoints (positions, heights) of the surface along a ray parallel to x (along = 0, at z = c) or z (along = 2, at
        x = c): every cell edge and every crossing of the cell diagonal."""
        if along == 0:
            i, v = self.cell(c, self.hz, self.dz, self.nr - 1)
            x = -self.hx + self.dx * np.arange(self.nc)
            e = self.H[i] + v * (self.H[i + 1] - self.H[i])
            fd = 1 - v if not self.zig else v
            if not self.zig:
                dg = self.H[i, 1:] + v * (self.H[i + 1, :-1] - self.H[i, 1:])
            else:
                dg = self.H[i, :-1] + v * (self.H[i + 1, 1:] - self.H[i, :-1])
            xd = x[:-1] + fd * self.dx
        else:
            j, u = self.cell(c, self.hx, self.dx, self.nc - 1)
            x = -self.hz + self.dz * np.arange(self.nr)
            e = self.H[:, j] + u * (self.H[:, j + 1] - self.H[:, j])
            fd = 1 - u if not self.zig else u
            if not self.zig:
                dg = self.H[1:, j] + u * (self.H[:-1, j + 1] - self.H[1:, j])
            else:
                dg = self.H[:-1, j] + u * (self.H[1:, j + 1] - self.H[:-1, j])
            xd = x[:-1] + fd * (self.dz)
        pos = np.empty(2 * len(x) - 1)
        val = np.empty(2 * len(x) - 1)
        pos[0::2], pos[1::2] = x, xd
        val[0::2], val[1::2] = e, dg
        return pos, val * self.sy


def crossings(shape, hf, i, cj, ck):
    """Crossings of the ray along axis i at (coordinate cj on axis (i + 1) % 3, ck on (i + 2) % 3), ascending, as (X, eX), and
    the position from which the ray is undecided (inf: nowhere, -inf: the whole ray)."""
    cj, ck = float(cj), float(ck)
    if shape.kind == BALL:
        r = float(shape.params[0])
        return _sqrt_pair(r * r - cj * cj - ck * ck, 4 * U * (r * r + cj * cj + ck * ck))
    if shape.kind == CUBOID:
        he = [float(p) for p in shape.params]
        j, k = (i + 1) % 3, (i + 2) % 3
        if abs(cj) <= he[j] and abs(ck) <= he[k]:
            return [(-he[i], 0.0), (he[i], 0.0)], math.inf
        return [], math.inf
    if shape.kind == CAPSULE:
        hh, r = float(shape.params[0]), float(shape.params[1])
        if i == 1:
            return _sqrt_pair(r * r - cj * cj - ck * ck, 4 * U * (r * r + cj * cj + ck * ck), hh, U * hh)
        y, c = (cj, ck) if i == 0 else (ck, cj)
        dy = max(abs(y) - hh, 0.0)
        return _sqrt_pair(r * r - dy * dy - c * c, 6 * U * (r * r + dy * dy + c * c))
    # heightfield
    if i == 1:
        x, z = ck, cj
        if not (-hf.hx <= x <= hf.hx and -hf.hz <= z <= hf.hz):
            return [], math.inf
        flat = hf.flat_cell(x, z)
        if flat is not None:  # inside a flat cell, clear of its edges: the device's height is fl(h * sy) exactly
            return [(float(F32(flat) * F32(hf.sy)), 0.0)], math.inf
        Y = hf.height(x, z)
        return [(Y, 2 * hf.Ef + 4 * U * abs(Y))], math.inf
    y, c = (cj, ck) if i == 0 else (ck, cj)
    half = hf.hz if i == 0 else hf.hx
    if not (-half <= c <= half):
        return [], math.inf
    pos, h = hf.profile(i, c)
    f = h - y
    Ef = hf.Ef + 4 * U * abs(y)
    near = np.nonzero(np.abs(f) <= Ef)[0]
    undec = math.inf
    if len(near):
        undec = float(pos[near[0]]) - hf.ex - (hf.ev + 4 * U) * max(hf.dx, hf.dz)  # a ray at a vertex height of its profile
    out = []
    neg = f < 0
    for s in np.nonzero(neg[:-1] != neg[1:])[0]:
        xa, xb, fa, fb = pos[s], pos[s + 1], f[s], f[s + 1]
        X = xa + (xb - xa) * fa / (fa - fb)
        eX = 2 * (hf.ex + (hf.ev + 2 * U) * max(hf.dx, hf.dz)) + abs(xb - xa) * (Ef / (abs(fa) + abs(fb)) + 4 * U) + 2 * U * abs(X)
        out.append((float(X), float(eX)))
    return out, undec


# -- the loops -----------------------------------------------------------------------------------------------------------
class Result:
    """Keys the reference decides (`keys`, sorted unique int64), keys it leaves undecided (`undecided`), and `lines`: (axis,
    key on axis (i + 1) % 3, key on (i + 2) % 3, first undecided key along the axis) for rays undecided from a point on."""

    def __init__(self, keys, undecided, lines, origin, sub, rays):
        self.keys, self.undecided, self.lines, self.origin, self.sub, self.rays = keys, undecided, lines, origin, sub, rays


def _u32(q):
    q = float(q)
    if not q > 0:
        return 0
    return min(int(q), 0xFFFFFFFF)


def _round(q):
    return F32(math.floor(abs(float(q)) + 0.5) * (1 if q >= 0 else -1))  # round half away from zero


def sample(shape, particle_rad, volume, bugs=()):
    """surface_ray_sample / volume_ray_sample (ray_sampling.rs:27-164) as a Result."""
    bugs = set(bugs)
    sub, sub10, origin, tabs = grid(shape, particle_rad, bugs)
    hf = _HF(shape, bugs) if shape.kind == HEIGHTFIELD else None
    keys, und, lines = [], [], []
    rays = 0

    def emit(c, dst):
        dst.append(key(c))

    for i in range(3):
        j, k = (i + 1) % 3, (i + 2) % 3
        for a, cj in enumerate(tabs[j]):
            for b, ck in enumerate(tabs[k]):
                if i > 0 and a == 0 and b == 0:
                    continue  # the first row of the y and z families starts one step in
                rays += 1
                qj, qk = (cj - origin[j]) / sub, (ck - origin[k]) / sub
                rnd = (lambda q: F32(math.floor(q))) if "floor_across" in bugs else _round
                kj, kk = _u32(rnd(qj)), _u32(rnd(qk))
                xs, undec_at = crossings(shape, hf, i, cj, ck)
                o_lo = o_hi = tabs[i][0]
                entry, prev = True, None
                cut = None  # first undecided along-key of the ray

                def put(along, dst):
                    c = [0, 0, 0]
                    c[i], c[j], c[k] = along, kj, kk
                    emit(c, dst)

                def quant(imp):
                    return (imp - origin[i]) / sub

                for X, eX in xs:
                    if X + eX >= undec_at:
                        cut = undec_at
                        break
                    Xlo, Xhi = _down(X - eX), _up(X + eX)
                    if Xlo >= o_hi:  # the cast from o finds X (toi >= 0)
                        ahead = True
                    elif Xhi < o_lo:
                        ahead = False
                    else:
                        cut = min(float(Xlo), float(o_lo))
                        break
                    if not ahead:
                        if "skip_keeps_parity" in bugs:
                            entry = not entry
                            prev = None if prev is not None else (quant(Xlo), quant(Xhi))
                        continue
                    if o_lo == o_hi:  # impact = o + (X - o) and the advance, both monotone in X
                        o = o_lo
                        toi_lo, toi_hi = F32(Xlo - o), F32(Xhi - o)
                        imp_lo, imp_hi = F32(o + toi_lo), F32(o + toi_hi)
                        n_lo, n_hi = F32(o + F32(toi_lo + sub10)), F32(o + F32(toi_hi + sub10))
                    else:
                        w = U * (abs(X) + abs(float(o_hi)) + abs(X - float(o_lo))) * 1.01
                        imp_lo, imp_hi = _down(X - eX - w), _up(X + eX + w)
                        w2 = U * (abs(X - float(o_lo)) + float(sub10) + abs(X + float(sub10))) * 2.02 + w
                        n_lo, n_hi = _down(X - eX + float(sub10) - w2), _up(X + eX + float(sub10) + w2)
                    if "no_skip" in bugs:  # only the crossings strictly after the impact remain
                        n_lo, n_hi = np.nextafter(imp_lo, F32(np.inf)), np.nextafter(imp_hi, F32(np.inf))
                    q_lo, q_hi = quant(imp_lo), quant(imp_hi)
                    if not volume:
                        use_ceil = entry != ("ceil_floor_swapped" in bugs)
                        fn = math.ceil if use_ceil else math.floor
                        c_lo, c_hi = _u32(fn(q_lo)), _u32(fn(q_hi))
                        for v in range(c_lo, c_hi + 1):
                            put(v, keys if c_lo == c_hi else und)
                    elif prev is None:
                        prev = (q_lo, q_hi)
                    else:
                        s_lo, s_hi = _u32(_round(prev[0])), _u32(_round(prev[1]))
                        e_lo, e_hi = _u32(_round(q_lo)), _u32(_round(q_hi))
                        if "exclusive_end" in bugs:
                            e_lo, e_hi = e_lo - 1, e_hi - 1
                        for v in range(s_lo, min(s_hi, e_hi + 1)):
                            put(v, und)
                        if s_hi <= e_lo:
                            lo = np.arange(s_hi, e_lo + 1, dtype=np.int64)
                            c = [None] * 3
                            c[i], c[j], c[k] = lo, np.int64(kj), np.int64(kk)
                            keys.extend(((c[0] << (2 * KEY_BITS)) | (c[1] << KEY_BITS) | c[2]).tolist())
                        for v in range(max(e_lo + 1, s_hi), e_hi + 1):
                            put(v, und)
                        prev = None
                    o_lo, o_hi = n_lo, n_hi
                    entry = not entry
                if cut is not None:
                    first = max(int(math.floor((cut - float(origin[i])) / float(sub))) - 1, 0)
                    lines.append((i, kj, kk, first))
    keys = np.unique(np.asarray(keys, np.int64))
    und = np.setdiff1d(np.unique(np.asarray(und, np.int64)), keys)
    return Result(keys, und, lines, origin, sub, rays)


def unquantize(keys, origin, sub, bugs=()):
    """unquantize_points ray_sampling.rs:193-207: origin + (e as f32) * sub, rounded after the multiply and after the add."""
    e = unkey(keys).astype(F32)
    if "fma_unquantize" in bugs:
        return (origin.astype(np.float64) + e.astype(np.float64) * np.float64(sub)).astype(F32)
    return (origin + e * sub).astype(F32)


def keys_of_points(points, origin, sub):
    """The keys of sampled points (the inverse of unquantize on its image)."""
    e = np.rint((np.asarray(points, np.float64) - origin.astype(np.float64)) / float(sub)).astype(np.int64)
    if len(e) and (e.min() < 0 or e.max() >= KEY_LIM):
        raise AssertionError("a point lies off the key grid")
    return (e[:, 0] << (2 * KEY_BITS)) | (e[:, 1] << KEY_BITS) | e[:, 2]


def compare(dev_keys, ref):
    """Checks a sampler's key set against the reference: every decided key present, every other key undecided.  Returns
    (missing decided keys, unexplained keys, undecided keys met) as counts."""
    dev = np.unique(np.asarray(dev_keys, np.int64))
    missing = np.setdiff1d(ref.keys, dev)
    extra = np.setdiff1d(dev, ref.keys)
    in_und = np.isin(extra, ref.undecided)
    rest = extra[~in_und]
    if len(rest) and ref.lines:
        c = unkey(rest)
        ok = np.zeros(len(rest), bool)
        for (i, kj, kk, first) in ref.lines:
            j, k = (i + 1) % 3, (i + 2) % 3
            ok |= (c[:, j] == kj) & (c[:, k] == kk) & (c[:, i] >= first)
        rest = rest[~ok]
    # decided keys on an undecided line's tail are decided only up to its cut
    if len(missing) and ref.lines:
        c = unkey(missing)
        ok = np.zeros(len(missing), bool)
        for (i, kj, kk, first) in ref.lines:
            j, k = (i + 1) % 3, (i + 2) % 3
            ok |= (c[:, j] == kj) & (c[:, k] == kk) & (c[:, i] >= first)
        missing = missing[~ok]
    return len(missing), len(rest), int(len(ref.undecided))


def cuboid_counts(n):
    """Closed-form key counts of a cuboid with half extents n[a] * particle_rad when every operation is exact (a dyadic
    particle_rad): the ray grid then lies half a cell off every face, entries quantise to 0.5 and exits to n + 0.5."""
    X, Y, Z = n
    volume = X * Y * Z + Y * Z + X * Z + X * Y
    surface = X * Y * Z - max(X - 2, 0) * max(Y - 2, 0) * max(Z - 2, 0)
    return surface, volume
