// sph_diffuse.cuh — diffuse particles: spray, foam and air bubbles (DESIGN.md section 16; host side in sph_diffuse_host.inl).
//
// A one-way post-process after Ihmsen et al. 2012: potentials of the binned fluid (sph_surface_host.inl bins_sort) decide how
// many diffuse particles each fluid particle emits; every diffuse particle is then classified by its fluid neighbour count
// and advected.  The neighbour loops are surf_for_cells' 27 cells in 9 z-runs over the binning's own grid; nothing here reads
// or writes the step's grid constants or arrays.  The float operations that decide a count or a kind are written out with
// explicit roundings, as include/sph.h states them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "sph_hash.h"

namespace sphk {

enum { DIFFUSE_SPRAY = 0, DIFFUSE_FOAM = 1, DIFFUSE_BUBBLE = 2 };

struct DiffuseParams {  // one update: sph_diffuse_desc and the call's arguments
    float ta_min, ta_max, wc_min, wc_max, k_min, k_max;
    float k_ta, k_wc, lifetime, k_b, k_d;
    float dt, g[3], lo[3], hi[3];
    float rp;                       // the world's particle radius
    uint32_t spray_below, bubble_above, seed, counter;
    float rho0[MAX_FLUIDS];         // per fluid slot
};

// min(a, b) as (b < a) ? b : a: a NaN first operand stays NaN
__device__ __forceinline__ float diffuse_min(float a, float b) { return b < a ? b : a; }
// Phi(I, lo, hi) = (min(I, hi) - min(I, lo)) / (hi - lo)
__device__ __forceinline__ float diffuse_clamp(float I, float lo, float hi) {
    return __fdiv_rn(__fsub_rn(diffuse_min(I, hi), diffuse_min(I, lo)), __fsub_rn(hi, lo));
}

// Normals of the binned fluid: n_i = -grad phi(x_i) / |grad phi(x_i)|, 0 where the gradient is 0 (k_surf_normals' rule).
__global__ void k_diffuse_normals(uint32_t n, SurfGrid g, const uint32_t* __restrict__ cstart, const float4* __restrict__ sp,
                                  float4* __restrict__ nrm) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const float4 p = sp[s];
    float4 acc;
    surf_gather<true>(p.x, p.y, p.z, g, cstart, sp, acc);
    const float n2 = dist2_exact(acc.x, acc.y, acc.z);
    const float sc = n2 > 0.f ? -__frsqrt_rn(n2) : 0.f;
    nrm[s] = make_float4(acc.x * sc, acc.y * sc, acc.z * sc, 0.f);
}

// Potentials and emission counts of the binned fluid.  Per sorted particle s: the trapped-air and wave-crest sums over the
// fluid within h, the kinetic energy and n_d; cnt[s] = n_d in cell order, the four values and the normal also at the
// particle's collected row perm[s].
__global__ void k_diffuse_potentials(uint32_t n, SurfGrid g, const uint32_t* __restrict__ cstart, const float4* __restrict__ sp,
                                     const float4* __restrict__ sv, const float4* __restrict__ nrm, const uint32_t* __restrict__ perm,
                                     const unsigned long long* __restrict__ key, DiffuseParams P, unsigned long long* __restrict__ cnt,
                                     float* __restrict__ o_nrm, float* __restrict__ o_ta, float* __restrict__ o_wc, float* __restrict__ o_ek,
                                     uint32_t* __restrict__ o_nd) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const float4 pi = sp[s], vi = sv[s], ni = nrm[s];
    float ta = 0.f, kap = 0.f;
    surf_for_cells(pi.x, pi.y, pi.z, g, cstart, [&](uint32_t j) {
        const float4 pj = sp[j];
        const float dx = __fsub_rn(pi.x, pj.x), dy = __fsub_rn(pi.y, pj.y), dz = __fsub_rn(pi.z, pj.z);
        const float d2 = dist2_exact(dx, dy, dz);
        if (!(d2 <= C.h2)) return;
        const float r = __fsqrt_rn(d2);
        const float wt = __fsub_rn(1.f, __fdiv_rn(r, C.h));  // W~(r) = 1 - r / h
        const float4 vj = sv[j];
        const float ux = __fsub_rn(vi.x, vj.x), uy = __fsub_rn(vi.y, vj.y), uz = __fsub_rn(vi.z, vj.z);
        const float vn = __fsqrt_rn(dist2_exact(ux, uy, uz));
        if (r > 0.f && vn > 0.f) {  // |v_ij| (1 - v^_ij . x^_ij) W~
            const float c = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(ux, dx), __fmul_rn(uy, dy)), __fmul_rn(uz, dz)), __fmul_rn(vn, r));
            ta = __fmaf_rn(__fmul_rn(vn, __fsub_rn(1.f, c)), wt, ta);
        }
        // (x_j - x_i) . n_i < 0, i.e. x_ij . n_i > 0: j lies behind the surface at i
        if (__fadd_rn(__fadd_rn(__fmul_rn(ni.x, dx), __fmul_rn(ni.y, dy)), __fmul_rn(ni.z, dz)) > 0.f) {
            const float4 nj = nrm[j];
            const float nn = __fadd_rn(__fadd_rn(__fmul_rn(ni.x, nj.x), __fmul_rn(ni.y, nj.y)), __fmul_rn(ni.z, nj.z));
            kap = __fmaf_rn(__fsub_rn(1.f, nn), wt, kap);
        }
    });
    const float v2 = dist2_exact(vi.x, vi.y, vi.z);
    const float vmag = __fsqrt_rn(v2);
    const float vdn = __fadd_rn(__fadd_rn(__fmul_rn(vi.x, ni.x), __fmul_rn(vi.y, ni.y)), __fmul_rn(vi.z, ni.z));
    const bool crest = vmag > 0.f && __fdiv_rn(vdn, vmag) >= 0.6f;  // v^_i . n_i >= 0.6
    const float wc = crest ? kap : 0.f;
    const unsigned long long kf = key[perm[s]];
    const uint32_t f = (uint32_t)(kf >> 32), id = (uint32_t)kf;
    const float ek = __fmul_rn(__fmul_rn(__fmul_rn(0.5f, pi.w), P.rho0[f]), v2);
    const float pta = diffuse_clamp(ta, P.ta_min, P.ta_max), pwc = diffuse_clamp(wc, P.wc_min, P.wc_max);
    const float pk = diffuse_clamp(ek, P.k_min, P.k_max);
    const float u = sph_hash_unit(sph_diffuse_hash(P.seed, P.counter, f, id, 0u, 0u));
    const float e = __fadd_rn(__fmul_rn(__fmul_rn(pk, __fadd_rn(__fmul_rn(P.k_ta, pta), __fmul_rn(P.k_wc, pwc))), P.dt), u);
    const uint32_t nd = e >= 1.f ? (e >= 4294967296.f ? 0xFFFFFFFFu : (uint32_t)e) : 0u;  // floor; NaN emits nothing
    cnt[s] = nd;
    const uint32_t o = perm[s];
    o_nrm[3 * (size_t)o] = ni.x;
    o_nrm[3 * (size_t)o + 1] = ni.y;
    o_nrm[3 * (size_t)o + 2] = ni.z;
    o_ta[o] = ta;
    o_wc[o] = wc;
    o_ek[o] = ek;
    o_nd[o] = nd;
}

// Emission: sorted fluid particle s emits its particles k = 0 .. cnt - 1 at rows base + off[s] + k, those below base + room.
// Each is sampled in the cylinder of radius r_p around v_f (Duff et al. 2017's basis) and dt |v_f| long.
__global__ void k_diffuse_emit(uint32_t n, const float4* __restrict__ sp, const float4* __restrict__ sv, const uint32_t* __restrict__ perm,
                               const unsigned long long* __restrict__ key, const unsigned long long* __restrict__ off, uint32_t base,
                               unsigned long long room, DiffuseParams P, float4* __restrict__ wx, float4* __restrict__ wv) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const unsigned long long o = off[s];
    if (o >= room) return;
    const unsigned long long m = min(off[s + 1] - o, room - o);
    if (!m) return;
    const unsigned long long kf = key[perm[s]];
    const uint32_t f = (uint32_t)(kf >> 32), id = (uint32_t)kf;
    const float4 xf = sp[s], vf = sv[s];
    const float speed = __fsqrt_rn(dist2_exact(vf.x, vf.y, vf.z));
    const float inv = speed > 0.f ? __fdiv_rn(1.f, speed) : 0.f;
    const float nx = vf.x * inv, ny = vf.y * inv, nz = vf.z * inv;
    const float sg = copysignf(1.f, nz);
    const float a = __fdiv_rn(-1.f, sg + nz);
    const float b = nx * ny * a;
    const float e1x = 1.f + sg * nx * nx * a, e1y = sg * b, e1z = -sg * nx;
    const float e2x = b, e2y = sg + ny * ny * a, e2z = -ny;
    for (uint32_t k = 0; k < (uint32_t)m; ++k) {
        const float xr = sph_hash_unit(sph_diffuse_hash(P.seed, P.counter, f, id, k, 1u));
        const float xt = sph_hash_unit(sph_diffuse_hash(P.seed, P.counter, f, id, k, 2u));
        const float xh = sph_hash_unit(sph_diffuse_hash(P.seed, P.counter, f, id, k, 3u));
        const float r = P.rp * sqrtf(xr);
        float sn, cs;
        sincosf(6.28318530717958647692f * xt, &sn, &cs);
        const float rc = r * cs, rs = r * sn, hdt = xh * P.dt;
        const float ox = rc * e1x + rs * e2x, oy = rc * e1y + rs * e2y, oz = rc * e1z + rs * e2z;
        const size_t row = base + o + k;
        wx[row] = make_float4(xf.x + ox + hdt * vf.x, xf.y + oy + hdt * vf.y, xf.z + oz + hdt * vf.z, P.lifetime);
        wv[row] = make_float4(vf.x + ox, vf.y + oy, vf.z + oz, 0.f);
    }
}

// Classification and advection of every diffuse particle: rows [0, n_old) from the last set, the rest as emitted into wx /
// wv.  Writes the advected particle back to wx / wv (kind in wv.w's bits) and keep[d]; counts the removals and the kinds of
// the survivors into totals (expired, left the box, spray, foam, bubble).
__global__ void k_diffuse_advect(uint32_t n, uint32_t n_old, const float* __restrict__ pos, const float* __restrict__ vel,
                                 const float* __restrict__ life, SurfGrid g, const uint32_t* __restrict__ cstart, const float4* __restrict__ sp,
                                 const float4* __restrict__ sv, DiffuseParams P, float4* __restrict__ wx, float4* __restrict__ wv,
                                 uint32_t* __restrict__ keep, unsigned long long* __restrict__ totals) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t counts[5] = {0u, 0u, 0u, 0u, 0u};
    if (d < n) {
        float x[3], v[3], lf;
        if (d < n_old) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                x[a] = pos[3 * (size_t)d + a];
                v[a] = vel[3 * (size_t)d + a];
            }
            lf = life[d];
        } else {
            const float4 p = wx[d], q = wv[d];
            x[0] = p.x, x[1] = p.y, x[2] = p.z, lf = p.w;
            v[0] = q.x, v[1] = q.y, v[2] = q.z;
        }
        uint32_t nn = 0;
        float sw = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f;
        const float x0 = x[0], x1 = x[1], x2 = x[2];
        if (isfinite(x0) && isfinite(x1) && isfinite(x2))
            surf_for_cells(x0, x1, x2, g, cstart, [&](uint32_t j) {
                const float4 pj = sp[j];
                const float d2 = dist2_exact(__fsub_rn(x0, pj.x), __fsub_rn(x1, pj.y), __fsub_rn(x2, pj.z));
                if (!(d2 <= C.h2)) return;
                ++nn;
                const float wgt = kernel_w_kind(C.kw, __fsqrt_rn(d2));
                const float4 vj = sv[j];
                sw = __fadd_rn(sw, wgt);
                s0 = __fmaf_rn(wgt, vj.x, s0);
                s1 = __fmaf_rn(wgt, vj.y, s1);
                s2 = __fmaf_rn(wgt, vj.z, s2);
            });
        const float s[3] = {s0, s1, s2};
        uint32_t kind;
        if (nn < P.spray_below) {
            kind = DIFFUSE_SPRAY;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                v[a] = __fmaf_rn(P.dt, P.g[a], v[a]);
                x[a] = __fmaf_rn(P.dt, v[a], x[a]);
            }
        } else {
            float vt[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) vt[a] = sw > 0.f ? __fdiv_rn(s[a], sw) : 0.f;
            if (nn > P.bubble_above) {
                kind = DIFFUSE_BUBBLE;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    v[a] = __fmaf_rn(P.k_d, __fsub_rn(vt[a], v[a]), __fsub_rn(v[a], __fmul_rn(__fmul_rn(P.dt, P.k_b), P.g[a])));
                    x[a] = __fmaf_rn(P.dt, v[a], x[a]);
                }
            } else {
                kind = DIFFUSE_FOAM;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    v[a] = vt[a];
                    x[a] = __fmaf_rn(P.dt, vt[a], x[a]);
                }
                lf = __fsub_rn(lf, P.dt);
            }
        }
        const bool expired = kind == DIFFUSE_FOAM && !(lf > 0.f);
        bool inside = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) inside &= P.lo[a] <= x[a] && x[a] < P.hi[a];  // NaN is outside
        const bool k = !expired && inside;
        counts[0] = expired;
        counts[1] = !expired && !inside;
        counts[2] = k && kind == DIFFUSE_SPRAY;
        counts[3] = k && kind == DIFFUSE_FOAM;
        counts[4] = k && kind == DIFFUSE_BUBBLE;
        wx[d] = make_float4(x[0], x[1], x[2], lf);
        wv[d] = make_float4(v[0], v[1], v[2], __uint_as_float(kind));
        keep[d] = k;
    }
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        const uint32_t t = __reduce_add_sync(0xffffffffu, counts[c]);
        if ((threadIdx.x & 31) == 0 && t) atomicAdd(&totals[c], (unsigned long long)t);
    }
}

// Compaction: the kept rows of wx / wv, in order, into the published layout (row = the exclusive scan of keep).
__global__ void k_diffuse_compact(uint32_t n, const uint32_t* __restrict__ row, const float4* __restrict__ wx, const float4* __restrict__ wv,
                                  float* __restrict__ pos, float* __restrict__ vel, uint8_t* __restrict__ kind, float* __restrict__ life) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n) return;
    const uint32_t o = row[d];
    if (row[d + 1] == o) return;
    const float4 p = wx[d], q = wv[d];
    pos[3 * (size_t)o] = p.x;
    pos[3 * (size_t)o + 1] = p.y;
    pos[3 * (size_t)o + 2] = p.z;
    vel[3 * (size_t)o] = q.x;
    vel[3 * (size_t)o + 1] = q.y;
    vel[3 * (size_t)o + 2] = q.z;
    kind[o] = (uint8_t)__float_as_uint(q.w);
    life[o] = p.w;
}

}  // namespace sphk
