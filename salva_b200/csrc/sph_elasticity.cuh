// sph_elasticity.cuh — Becker2009 corotated SPH elasticity (becker2009_elasticity.rs:84-334).
//
// The rest pose (positions0, volumes0, contacts0) is keyed by ORIGINAL particle index (the reference's lists are
// fixed when the force is first solved, :84-113), so these kernels run in the fluid's original index space
// t = original index - fluid offset: current positions are first scattered to original order, the corotated
// force is accumulated there and added to the sorted acceleration array through slot_of[].
#pragma once
#include "sph_passes.cuh"

namespace sphk {

struct M3 {
    float m[3][3];
};
__device__ __forceinline__ float3 m3_mul(const M3& a, float3 v) {
    return make_float3(a.m[0][0] * v.x + a.m[0][1] * v.y + a.m[0][2] * v.z, a.m[1][0] * v.x + a.m[1][1] * v.y + a.m[1][2] * v.z,
                       a.m[2][0] * v.x + a.m[2][1] * v.y + a.m[2][2] * v.z);
}
__device__ __forceinline__ float3 m3_tmul(const M3& a, float3 v) {
    return make_float3(a.m[0][0] * v.x + a.m[1][0] * v.y + a.m[2][0] * v.z, a.m[0][1] * v.x + a.m[1][1] * v.y + a.m[2][1] * v.z,
                       a.m[0][2] * v.x + a.m[1][2] * v.y + a.m[2][2] * v.z);
}
__device__ __forceinline__ M3 m3_load(const float* p) {
    M3 r;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) r.m[a][b] = p[a * 3 + b];
    return r;
}
__device__ __forceinline__ void m3_store(float* p, const M3& r) {
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) p[a * 3 + b] = r.m[a][b];
}
__device__ __forceinline__ float3 cross3(float3 a, float3 b) { return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// scatter the fluid's particles to original order: cur[t] = (pos.xyz, mass), slot_of[t] = s
__global__ void k_el_to_orig(const float4* __restrict__ pos, const uint32_t* __restrict__ orig, uint32_t lo, uint32_t hi, float4* __restrict__ cur,
                             uint32_t* __restrict__ slot_of) {
    SPH_OWNED_INDEX(s)
    uint32_t g = orig[s];
    if (g < lo || g >= hi) return;
    cur[g - lo] = pos[s];
    slot_of[g - lo] = s;
}

// rest contacts = this step's same-fluid contacts translated to original indices (compute_self_contacts contacts.rs:403-446
// on positions0 == current positions gives exactly the same set: same d^2 <= h^2 test, self included)
__global__ void k_el_capture_lists(Lists L, const float4* __restrict__ vel, const uint32_t* __restrict__ orig, const uint32_t* __restrict__ slot_of, uint32_t lo,
                                   uint32_t n, uint32_t which, uint32_t cap0, uint32_t stride0, uint32_t* __restrict__ nbr0, uint32_t* __restrict__ cnt0,
                                   uint32_t* __restrict__ maxcnt) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t i = slot_of[t];
    uint32_t cnt = L.fluid_count(i);
    uint32_t k0 = 0;
    for (uint32_t k = 0; k < cnt; ++k) {
        uint32_t j = L.fluid(i, k);
        if (fid_of(vel[j]) != which) continue;
        if (k0 < cap0) nbr0[(size_t)k0 * stride0 + t] = orig[j] - lo;
        ++k0;
    }
    cnt0[t] = k0;
    atomicMax(maxcnt, k0);
}

// positions0 + volumes0 (becker2009_elasticity.rs:89-111): vol0_i = m_i / (old_i + 2 * sum_j m_j W0_ij)
__global__ void k_el_rest_volumes(uint32_t n, const float4* __restrict__ cur, const uint32_t* __restrict__ nbr0, const uint32_t* __restrict__ cnt0,
                                  uint32_t stride0, const float* __restrict__ old_vol0, uint32_t old_n, float4* __restrict__ pos0) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    float4 pi = cur[t];
    float acc = 0.f;
    uint32_t cnt = cnt0[t];
    for (uint32_t k = 0; k < cnt; ++k) {
        uint32_t j = nbr0[(size_t)k * stride0 + t];
        float4 pj = cur[j];
        Pair p = make_pair<true, false, true>(pi, pj);
        // contact (t, j) adds m_j W to vol0[t]; its mirror (j, t) in j's list adds m_j W to vol0[t] again (:105-108)
        acc += 2.0f * pj.w * p.w;
    }
    float base = (old_vol0 && t < old_n) ? old_vol0[t] : 0.f;  // Vec::resize keeps the old leading values (:90)
    pos0[t] = make_float4(pi.x, pi.y, pi.z, pi.w / (base + acc));
}

// nalgebra 0.33 Rotation3::from_matrix_eps (Müller et al. 2016), restated like the oracle (PARITY UNPINNED upstream)
__device__ __forceinline__ M3 rot_from_scaled_axis(float3 aa) {
    float angle = sqrtf(dot3(aa, aa));
    M3 r;
    if (angle == 0.f) {
        r = M3{{{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}}};
        return r;
    }
    float3 u = make_float3(aa.x / angle, aa.y / angle, aa.z / angle);
    float s = sinf(angle), c = cosf(angle), t = 1.f - c;
    r.m[0][0] = u.x * u.x * t + c;       r.m[0][1] = u.x * u.y * t - u.z * s; r.m[0][2] = u.x * u.z * t + u.y * s;
    r.m[1][0] = u.x * u.y * t + u.z * s; r.m[1][1] = u.y * u.y * t + c;       r.m[1][2] = u.y * u.z * t - u.x * s;
    r.m[2][0] = u.x * u.z * t - u.y * s; r.m[2][1] = u.y * u.z * t + u.x * s; r.m[2][2] = u.z * u.z * t + c;
    return r;
}

// compute_rotations becker2009_elasticity.rs:115-137
__global__ void __launch_bounds__(128)
k_el_rotations(uint32_t n, const float4* __restrict__ cur, const float4* __restrict__ pos0, const uint32_t* __restrict__ nbr0, const uint32_t* __restrict__ cnt0,
               uint32_t stride0, float* __restrict__ rot) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    float4 pi = cur[t], qi = pos0[t];
    M3 a;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) a.m[r][c] = 0.f;
    uint32_t cnt = cnt0[t];
    for (uint32_t k = 0; k < cnt; ++k) {
        uint32_t j = nbr0[(size_t)k * stride0 + t];
        float4 pj = cur[j], qj = pos0[j];
        Pair rp = make_pair<true, false, true>(qi, qj);  // contact.weight at the rest pose
        float coeff = rp.w * pj.w;
        float3 p = make_float3(pj.x - pi.x, pj.y - pi.y, pj.z - pi.z);
        float3 q = make_float3((qj.x - qi.x) * coeff, (qj.y - qi.y) * coeff, (qj.z - qi.z) * coeff);
        a.m[0][0] += p.x * q.x; a.m[0][1] += p.x * q.y; a.m[0][2] += p.x * q.z;
        a.m[1][0] += p.y * q.x; a.m[1][1] += p.y * q.y; a.m[1][2] += p.y * q.z;
        a.m[2][0] += p.z * q.x; a.m[2][1] += p.z * q.y; a.m[2][2] += p.z * q.z;
    }
    M3 r = m3_load(rot + 9 * (size_t)t);
    for (int it = 0; it < 20; ++it) {
        float3 r0 = make_float3(r.m[0][0], r.m[1][0], r.m[2][0]), r1 = make_float3(r.m[0][1], r.m[1][1], r.m[2][1]),
               r2 = make_float3(r.m[0][2], r.m[1][2], r.m[2][2]);
        float3 a0 = make_float3(a.m[0][0], a.m[1][0], a.m[2][0]), a1 = make_float3(a.m[0][1], a.m[1][1], a.m[2][1]),
               a2 = make_float3(a.m[0][2], a.m[1][2], a.m[2][2]);
        float3 c0 = cross3(r0, a0), c1 = cross3(r1, a1), c2 = cross3(r2, a2);
        float3 axis = make_float3(c0.x + c1.x + c2.x, c0.y + c1.y + c2.y, c0.z + c1.z + c2.z);
        float denom = dot3(r0, a0) + dot3(r1, a1) + dot3(r2, a2);
        float sc = 1.0f / (fabsf(denom) + F32_EPS);
        float3 aa = make_float3(axis.x * sc, axis.y * sc, axis.z * sc);
        if (!(dot3(aa, aa) > F32_EPS * F32_EPS)) break;
        M3 d = rot_from_scaled_axis(aa);
        M3 nr;
#pragma unroll
        for (int x = 0; x < 3; ++x)
#pragma unroll
            for (int y = 0; y < 3; ++y) nr.m[x][y] = d.m[x][0] * r.m[0][y] + d.m[x][1] * r.m[1][y] + d.m[x][2] * r.m[2][y];
        r = nr;
    }
    m3_store(rot + 9 * (size_t)t, r);
}

// compute_stresses becker2009_elasticity.rs:139-262 (dim3)
__global__ void __launch_bounds__(128)
k_el_stresses(uint32_t n, const float4* __restrict__ cur, const float4* __restrict__ pos0, const uint32_t* __restrict__ nbr0, const uint32_t* __restrict__ cnt0,
              uint32_t stride0, const float* __restrict__ rot, float* __restrict__ grad_tr, float* __restrict__ stress, float d0, float d1, float d2,
              int nonlinear) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    float4 pi = cur[t], qi = pos0[t];
    M3 R = m3_load(rot + 9 * (size_t)t);
    M3 g;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) g.m[r][c] = 0.f;
    uint32_t cnt = cnt0[t];
    for (uint32_t k = 0; k < cnt; ++k) {
        uint32_t j = nbr0[(size_t)k * stride0 + t];
        float4 pj = cur[j], qj = pos0[j];
        Pair rp = make_pair<false, true, true>(qi, qj);  // contact.gradient at the rest pose = rp.g * (q_i - q_j)
        float3 p = make_float3(pj.x - pi.x, pj.y - pi.y, pj.z - pi.z);
        float3 u = m3_tmul(R, p);  // inverse_transform_vector
        u.x -= qj.x - qi.x; u.y -= qj.y - qi.y; u.z -= qj.z - qi.z;
        float sc = rp.g * qj.w;  // gradient * volumes0[j]
        float3 a = make_float3(sc * rp.dx, sc * rp.dy, sc * rp.dz);
        g.m[0][0] += a.x * u.x; g.m[0][1] += a.x * u.y; g.m[0][2] += a.x * u.z;
        g.m[1][0] += a.y * u.x; g.m[1][1] += a.y * u.y; g.m[1][2] += a.y * u.z;
        g.m[2][0] += a.z * u.x; g.m[2][1] += a.z * u.y; g.m[2][2] += a.z * u.z;
    }
    m3_store(grad_tr + 9 * (size_t)t, g);
    const float kk = 0.564f;  // sic: the constant the reference names _0_5 (:141)
    float* s = stress + 6 * (size_t)t;
    if (nonlinear) {
        M3 J = g;
        J.m[0][0] += 1.f; J.m[1][1] += 1.f; J.m[2][2] += 1.f;
        float jj[3][3];
#pragma unroll
        for (int x = 0; x < 3; ++x)
#pragma unroll
            for (int y = 0; y < 3; ++y) jj[x][y] = J.m[x][0] * J.m[y][0] + J.m[x][1] * J.m[y][1] + J.m[x][2] * J.m[y][2];
        float ex = jj[0][0] - 1.f, ey = jj[1][1] - 1.f, ez = jj[2][2] - 1.f;
        s[0] = (d0 * ex + d1 * ey + d1 * ez) * kk;
        s[1] = (d1 * ex + d0 * ey + d1 * ez) * kk;
        s[2] = (d1 * ex + d1 * ey + d0 * ez) * kk;
        s[3] = jj[1][0] * kk * d2;
        s[4] = jj[2][0] * kk * d2;
        s[5] = jj[2][1] * kk * d2;
    } else {
        float ex = g.m[0][0], ey = g.m[1][1], ez = g.m[2][2];
        s[0] = d0 * ex + d1 * ey + d1 * ez;
        s[1] = d1 * ex + d0 * ey + d1 * ez;
        s[2] = d1 * ex + d1 * ey + d0 * ez;
        s[3] = (g.m[1][0] + g.m[0][1]) * kk * d2;
        s[4] = (g.m[2][0] + g.m[0][2]) * kk * d2;
        s[5] = (g.m[1][2] + g.m[2][1]) * kk * d2;
    }
}

__device__ __forceinline__ float3 sym_mul(const float* s, float3 v) {  // :27-37
    return make_float3(s[0] * v.x + s[3] * v.y + s[4] * v.z, s[3] * v.x + s[1] * v.y + s[5] * v.z, s[4] * v.x + s[5] * v.y + s[2] * v.z);
}

// forces becker2009_elasticity.rs:268-334: acceleration_i += 0.5 (R_j f_ij - R_i f_ji) / m_i over the rest contacts
__global__ void __launch_bounds__(128)
k_el_forces(uint32_t n, const float4* __restrict__ cur, const float4* __restrict__ pos0, const uint32_t* __restrict__ nbr0, const uint32_t* __restrict__ cnt0,
            uint32_t stride0, const float* __restrict__ rot, const float* __restrict__ grad_tr, const float* __restrict__ stress,
            const uint32_t* __restrict__ slot_of, float4* __restrict__ acc, int nonlinear) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    float4 qi = pos0[t];
    float mi = cur[t].w;
    M3 Ri = m3_load(rot + 9 * (size_t)t);
    M3 Gi = m3_load(grad_tr + 9 * (size_t)t);
    float si[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) si[a] = stress[6 * (size_t)t + a];
    float ax = 0.f, ay = 0.f, az = 0.f;
    uint32_t cnt = cnt0[t];
    for (uint32_t k = 0; k < cnt; ++k) {
        uint32_t j = nbr0[(size_t)k * stride0 + t];
        float4 qj = pos0[j];
        Pair rp = make_pair<false, true, true>(qi, qj);
        float3 grad = make_float3(rp.g * rp.dx, rp.g * rp.dy, rp.g * rp.dz);
        float3 d_ij = make_float3(grad.x * qj.w, grad.y * qj.w, grad.z * qj.w);
        float3 sd_ij = sym_mul(si, d_ij);
        float sj[6];
#pragma unroll
        for (int a = 0; a < 6; ++a) sj[a] = stress[6 * (size_t)j + a];
        float3 d_ji = make_float3(-grad.x * qi.w, -grad.y * qi.w, -grad.z * qi.w);
        float3 sd_ji = sym_mul(sj, d_ji);
        float3 f_ji, f_ij;
        if (nonlinear) {
            M3 Gj = m3_load(grad_tr + 9 * (size_t)j);
            float3 gi = m3_mul(Gi, sd_ij), gj = m3_mul(Gj, sd_ji);
            f_ji = make_float3((sd_ij.x + gi.x) * -qi.w, (sd_ij.y + gi.y) * -qi.w, (sd_ij.z + gi.z) * -qi.w);
            f_ij = make_float3((sd_ji.x + gj.x) * -qj.w, (sd_ji.y + gj.y) * -qj.w, (sd_ji.z + gj.z) * -qj.w);
        } else {
            f_ji = make_float3(sd_ij.x * -qi.w, sd_ij.y * -qi.w, sd_ij.z * -qi.w);
            f_ij = make_float3(sd_ji.x * -qj.w, sd_ji.y * -qj.w, sd_ji.z * -qj.w);
        }
        M3 Rj = m3_load(rot + 9 * (size_t)j);
        float3 a = m3_mul(Rj, f_ij), b = m3_mul(Ri, f_ji);
        ax += (a.x - b.x) * 0.5f / mi;
        ay += (a.y - b.y) * 0.5f / mi;
        az += (a.z - b.z) * 0.5f / mi;
    }
    uint32_t s = slot_of[t];
    float4 A = acc[s];
    A.x += ax; A.y += ay; A.z += az;
    acc[s] = A;
}

__global__ void k_el_identity(uint32_t n, uint32_t from, float* __restrict__ rot) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x + from;
    if (t >= n) return;
    float* r = rot + 9 * (size_t)t;
    r[0] = 1.f; r[1] = 0.f; r[2] = 0.f; r[3] = 0.f; r[4] = 1.f; r[5] = 0.f; r[6] = 0.f; r[7] = 0.f; r[8] = 1.f;
}

}  // namespace sphk
