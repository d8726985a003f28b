// Ray sampling of shapes into particles: salva3d::sampling::shape_surface_ray_sample / shape_volume_ray_sample
// (sampling/ray_sampling.rs:9-231, 3-D branch), restated for the device.  DESIGN.md section 11.
//
// The host builds the loosened AABB, `origin` and the three per-axis tables of ray coordinates from the same f32 running
// sums as the reference (curr[k] += sub while curr[k] < maxs[k]).  Ray family i (rays along axis i) has its rows along
// j = (i + 1) % 3 and its columns along k = (i + 2) % 3; the first row of families 1 and 2 starts one step in, because the
// reference's traversal does not reset that coordinate before its first row.
//
// Every ray is an axis-aligned line, so its crossings with the shape have closed forms: two for a ball, cuboid, capsule,
// cylinder or cone (the cone's vertical pair, base and slant, is not symmetric), and for a heightfield a walk over the cells of the row (or column) strip the ray lies in, where the surface along the
// ray is a polyline with a break on every cell edge and on every cell diagonal.  Each ray then runs the reference's loop:
// the first crossing at or after the ray origin is the hit, impact = o + toi, the origin moves to o + (toi + sub / 10) and
// entry / exit alternate.  k_sample_rays runs twice with the same code: once to count each ray's keys, once (after a scan)
// to write them.  Keys are 21 bits per axis, x in the high bits, so ascending keys are the (x, y, z) lexicographic order.
#pragma once
#include <cstdint>

#include "sph_shapes.cuh"

namespace sphk {

enum { SMP_KEY_BITS = 21 };
constexpr uint32_t SMP_KEY_LIM = 1u << SMP_KEY_BITS;
constexpr unsigned long long SMP_KEY_MASK = SMP_KEY_LIM - 1;

struct SampleRays {
    int kind, volume;
    float p[4];                    // ball / cuboid / capsule / cylinder / cone parameters (sph_shape.p)
    float origin[3], sub, sub10;   // volume.mins + sub / 2, 2 * particle_rad, sub / 10
    const float* tab[3];           // ray coordinates along each axis (f32 running sums from origin)
    uint32_t n[3];                 // their counts
    unsigned long long fam_end[3]; // cumulative ray counts of families 0, 1, 2
    HfGrid hf;                     // heightfield: heights and grid constants (the closest-point search's cap, margin and dmin unused)
};

// `f64 as u32` of an integral f32: saturating, NaN -> 0
__device__ __forceinline__ uint32_t smp_u32(float q) {
    if (!(q > 0.f)) return 0u;
    if (q >= 4294967296.f) return 0xFFFFFFFFu;
    return (uint32_t)q;
}

struct SmpSink {
    unsigned long long* keys;  // nullptr: count only
    unsigned long long base, count;
    int* overflow;
    int i, j, k;
    uint32_t kj, kk;
    __device__ __forceinline__ void put(uint32_t along) {
        if (along >= SMP_KEY_LIM || kj >= SMP_KEY_LIM || kk >= SMP_KEY_LIM) {
            *overflow = 1;
            return;
        }
        if (keys)  // axis a sits at bit (2 - a) * 21
            keys[base + count] = ((unsigned long long)along << ((2 - i) * SMP_KEY_BITS)) | ((unsigned long long)kj << ((2 - j) * SMP_KEY_BITS)) |
                                 ((unsigned long long)kk << ((2 - k) * SMP_KEY_BITS));
        ++count;
    }
    // sample_segment ray_sampling.rs:166-191: start..=end
    __device__ __forceinline__ void put_range(uint32_t a, uint32_t b) {
        if (b < a) return;
        if (b >= SMP_KEY_LIM || kj >= SMP_KEY_LIM || kk >= SMP_KEY_LIM) {
            *overflow = 1;
            return;
        }
        if (!keys) {
            count += (unsigned long long)(b - a) + 1;
            return;
        }
        for (uint32_t e = a;; ++e) {
            put(e);
            if (e == b) break;
        }
    }
};

// perform_cast ray_sampling.rs:40-53 (surface) and :103-127 (volume), fed with the ray's crossings in ascending order
struct SmpWalk {
    float o, org, sub, sub10;
    int volume;
    bool entry, have_prev;
    float qprev;
    __device__ __forceinline__ void hit(float X, SmpSink& s) {
        if (!(X >= o)) return;  // behind the origin: passed over by an earlier advance
        const float toi = __fsub_rn(X, o);
        const float imp = __fadd_rn(o, toi);  // ray.point_at(toi)
        const float q = __fdiv_rn(__fsub_rn(imp, org), sub);
        if (!volume) {
            s.put(smp_u32(entry ? ceilf(q) : floorf(q)));  // quantize_point :209-231
        } else if (!have_prev) {
            qprev = q;
            have_prev = true;
        } else {
            s.put_range(smp_u32(roundf(qprev)), smp_u32(roundf(q)));
            have_prev = false;
        }
        o = __fadd_rn(o, __fadd_rn(toi, sub10));
        entry = !entry;
    }
};

__device__ __forceinline__ float smp_lerp(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// one linear piece of the surface along the ray: a crossing where the height above the ray changes sign (0 counts as above)
__device__ __forceinline__ void smp_piece(float xa, float xb, float fa, float fb, SmpWalk& wk, SmpSink& s) {
    if ((fa < 0.f) == (fb < 0.f)) return;
    wk.hit(__fadd_rn(xa, __fmul_rn(__fsub_rn(xb, xa), __fdiv_rn(fa, __fsub_rn(fa, fb)))), s);
}

// heightfield, ray along x at (y, z): the profile of cell row i at z fraction v.  In each cell the ray crosses triangle
// (p00, p10, p01) up to the diagonal at x0 + (1 - v) dx, then (p10, p11, p01).
__device__ void smp_hf_along_x(const SampleRays& P, float y, float z, SmpWalk& wk, SmpSink& s) {
    if (!(z >= -P.hf.hz && z <= P.hf.hz)) return;
    float v;
    const int i = smp_cell(z, P.hf.hz, P.hf.dz, P.hf.nrows - 1, &v);
    const float w1 = __fsub_rn(1.f, v);
    const float* r0 = P.hf.hgt + (size_t)i * P.hf.ncols;
    const float* r1 = r0 + P.hf.ncols;
    float xa = -P.hf.hx;
    float fa = __fsub_rn(__fmul_rn(smp_lerp(r0[0], r1[0], v), P.hf.sy), y);
    for (int c = 0; c + 1 < P.hf.ncols; ++c) {
        const float xb = smp_grid(c + 1, P.hf.ncols - 1, P.hf.hx, P.hf.dx);
        const float xd = __fadd_rn(xa, __fmul_rn(w1, P.hf.dx));
        const float fd = __fsub_rn(__fmul_rn(smp_lerp(r0[c + 1], r1[c], v), P.hf.sy), y);
        const float fb = __fsub_rn(__fmul_rn(smp_lerp(r0[c + 1], r1[c + 1], v), P.hf.sy), y);
        smp_piece(xa, xd, fa, fd, wk, s);
        smp_piece(xd, xb, fd, fb, wk, s);
        xa = xb;
        fa = fb;
    }
}

// heightfield, ray along z at (x, y): the profile of cell column j at x fraction u; the diagonal lies at z0 + (1 - u) dz
__device__ void smp_hf_along_z(const SampleRays& P, float x, float y, SmpWalk& wk, SmpSink& s) {
    if (!(x >= -P.hf.hx && x <= P.hf.hx)) return;
    float u;
    const int j = smp_cell(x, P.hf.hx, P.hf.dx, P.hf.ncols - 1, &u);
    const float w1 = __fsub_rn(1.f, u);
    const float* H = P.hf.hgt + j;
    const int nc = P.hf.ncols;
    float za = -P.hf.hz;
    float fa = __fsub_rn(__fmul_rn(smp_lerp(H[0], H[1], u), P.hf.sy), y);
    for (int r = 0; r + 1 < P.hf.nrows; ++r) {
        const float* h0 = H + (size_t)r * nc;
        const float* h1 = h0 + nc;
        const float zb = smp_grid(r + 1, P.hf.nrows - 1, P.hf.hz, P.hf.dz);
        const float zd = __fadd_rn(za, __fmul_rn(w1, P.hf.dz));
        const float fd = __fsub_rn(__fmul_rn(smp_lerp(h1[0], h0[1], u), P.hf.sy), y);
        const float fb = __fsub_rn(__fmul_rn(smp_lerp(h1[0], h1[1], u), P.hf.sy), y);
        smp_piece(za, zd, fa, fd, wk, s);
        smp_piece(zd, zb, fd, fb, wk, s);
        za = zb;
        fa = fb;
    }
}

// heightfield, ray along y at (x, z): one crossing at the surface height over the footprint
__device__ void smp_hf_along_y(const SampleRays& P, float x, float z, SmpWalk& wk, SmpSink& s) {
    if (!(x >= -P.hf.hx && x <= P.hf.hx && z >= -P.hf.hz && z <= P.hf.hz)) return;
    float u, v;
    const int j = smp_cell(x, P.hf.hx, P.hf.dx, P.hf.ncols - 1, &u);
    const int i = smp_cell(z, P.hf.hz, P.hf.dz, P.hf.nrows - 1, &v);
    const float* r0 = P.hf.hgt + (size_t)i * P.hf.ncols + j;
    const float* r1 = r0 + P.hf.ncols;
    const float h00 = r0[0], h10 = r0[1], h01 = r1[0], h11 = r1[1];  // h10: (x1, z0), h01: (x0, z1)
    float h;
    if (__fadd_rn(u, v) <= 1.f)
        h = __fadd_rn(__fadd_rn(h00, __fmul_rn(u, __fsub_rn(h10, h00))), __fmul_rn(v, __fsub_rn(h01, h00)));
    else
        h = __fadd_rn(__fadd_rn(h11, __fmul_rn(__fsub_rn(1.f, u), __fsub_rn(h01, h11))), __fmul_rn(__fsub_rn(1.f, v), __fsub_rn(h10, h11)));
    wk.hit(__fmul_rn(h, P.hf.sy), s);
}

__device__ __forceinline__ void smp_pair(float t, SmpWalk& wk, SmpSink& s) {
    wk.hit(-t, s);
    wk.hit(t, s);
}

// FILL == false: cnt[r] = number of keys of ray r; FILL == true: write them from off[r]
template <bool FILL>
__global__ void __launch_bounds__(256) k_sample_rays(SampleRays P, unsigned long long* cnt, const unsigned long long* off,
                                                     unsigned long long* keys, int* overflow) {
    const unsigned long long r = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (r >= P.fam_end[2]) return;
    const int i = r < P.fam_end[0] ? 0 : r < P.fam_end[1] ? 1 : 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    const unsigned long long lr = r - (i ? P.fam_end[i - 1] : 0ull);
    const uint32_t a = (uint32_t)(lr / P.n[k]), b = (uint32_t)(lr % P.n[k]);
    SmpSink s;
    s.keys = FILL ? keys : nullptr;
    s.base = FILL ? off[r] : 0ull;
    s.count = 0;
    s.overflow = overflow;
    s.i = i;
    s.j = j;
    s.k = k;
    if (!(i > 0 && a == 0 && b == 0)) {
        const float cj = P.tab[j][a], ck = P.tab[k][b];
        s.kj = smp_u32(roundf(__fdiv_rn(__fsub_rn(cj, P.origin[j]), P.sub)));
        s.kk = smp_u32(roundf(__fdiv_rn(__fsub_rn(ck, P.origin[k]), P.sub)));
        SmpWalk wk;
        wk.o = P.tab[i][0];
        wk.org = P.origin[i];
        wk.sub = P.sub;
        wk.sub10 = P.sub10;
        wk.volume = P.volume;
        wk.entry = true;
        wk.have_prev = false;
        wk.qprev = 0.f;
        const float r2 = __fmul_rn(P.p[1], P.p[1]);
        switch (P.kind) {
            case SPH_SHAPE_BALL: {
                const float sq = __fsub_rn(__fmul_rn(P.p[0], P.p[0]), __fadd_rn(__fmul_rn(cj, cj), __fmul_rn(ck, ck)));
                if (sq >= 0.f) smp_pair(__fsqrt_rn(sq), wk, s);
                break;
            }
            case SPH_SHAPE_CUBOID:  // closed
                if (fabsf(cj) <= P.p[j] && fabsf(ck) <= P.p[k]) smp_pair(P.p[i], wk, s);
                break;
            case SPH_SHAPE_CAPSULE: {  // segment [-p0, p0] along y, radius p1
                if (i == 1) {
                    const float sq = __fsub_rn(r2, __fadd_rn(__fmul_rn(cj, cj), __fmul_rn(ck, ck)));
                    if (sq >= 0.f) smp_pair(__fadd_rn(P.p[0], __fsqrt_rn(sq)), wk, s);
                } else {
                    const float y = i == 0 ? cj : ck, c = i == 0 ? ck : cj;
                    const float dy = fmaxf(__fsub_rn(fabsf(y), P.p[0]), 0.f);
                    const float sq = __fsub_rn(r2, __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(c, c)));
                    if (sq >= 0.f) smp_pair(__fsqrt_rn(sq), wk, s);
                }
                break;
            }
            case SPH_SHAPE_CYLINDER: {  // |y| <= p0, x^2 + z^2 <= p1^2, closed
                if (i == 1) {
                    if (__fsub_rn(r2, __fadd_rn(__fmul_rn(cj, cj), __fmul_rn(ck, ck))) >= 0.f) smp_pair(P.p[0], wk, s);
                } else {
                    const float y = i == 0 ? cj : ck, c = i == 0 ? ck : cj;
                    const float sq = __fsub_rn(r2, __fmul_rn(c, c));
                    if (fabsf(y) <= P.p[0] && sq >= 0.f) smp_pair(__fsqrt_rn(sq), wk, s);
                }
                break;
            }
            case SPH_SHAPE_CONE: {  // apex (0, p0, 0), base disc of radius p1 at y = -p0; radius R(y) = p1 (p0 - y) / (2 p0)
                const float a = P.p[0], a2 = __fadd_rn(a, a);
                if (i == 1) {  // the base, then the slant at y = a - 2a rho / r (a at rho = 0, -a at the rim)
                    const float c2 = __fadd_rn(__fmul_rn(cj, cj), __fmul_rn(ck, ck));
                    if (__fsub_rn(r2, c2) >= 0.f) {
                        const float rho = __fsqrt_rn(c2);
                        const float f = rho == 0.f ? 0.f : fminf(__fdiv_rn(rho, P.p[1]), 1.f);
                        wk.hit(-a, s);
                        wk.hit(__fsub_rn(a, __fmul_rn(a2, f)), s);
                    }
                } else {
                    const float y = i == 0 ? cj : ck, c = i == 0 ? ck : cj;
                    if (fabsf(y) <= a) {
                        const float R = a == 0.f ? P.p[1] : __fdiv_rn(__fmul_rn(P.p[1], __fsub_rn(a, y)), a2);
                        const float sq = __fsub_rn(__fmul_rn(R, R), __fmul_rn(c, c));
                        if (sq >= 0.f) smp_pair(__fsqrt_rn(sq), wk, s);
                    }
                }
                break;
            }
            default:  // heightfield
                if (i == 0) smp_hf_along_x(P, cj, ck, wk, s);
                else if (i == 1) smp_hf_along_y(P, ck, cj, wk, s);
                else smp_hf_along_z(P, cj, ck, wk, s);
        }
    }
    if (!FILL) cnt[r] = s.count;
}

// unquantize_points ray_sampling.rs:193-207: origin + (e as f32) * sub, one rounded multiply and one rounded add
__global__ void __launch_bounds__(256) k_sample_unquantize(const unsigned long long* keys, unsigned long long n, float ox, float oy,
                                                           float oz, float sub, float* xyz) {
    const unsigned long long m = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
    if (m >= n) return;
    const unsigned long long key = keys[m];
    xyz[3 * m + 0] = __fadd_rn(ox, __fmul_rn((float)(uint32_t)((key >> (2 * SMP_KEY_BITS)) & SMP_KEY_MASK), sub));
    xyz[3 * m + 1] = __fadd_rn(oy, __fmul_rn((float)(uint32_t)((key >> SMP_KEY_BITS) & SMP_KEY_MASK), sub));
    xyz[3 * m + 2] = __fadd_rn(oz, __fmul_rn((float)(uint32_t)(key & SMP_KEY_MASK), sub));
}

}  // namespace sphk
