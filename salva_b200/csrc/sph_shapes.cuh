// sph_shapes.cuh — shapes and colliders on the device: the parry geometry (heightfield, solids of revolution, the ball /
// cuboid / capsule projections), the shape and AABB point query, and the collider coupling kernels (static poses,
// impulses, DynamicContactSampling).  DESIGN.md sections 10 and 11.  The host side is sph_colliders_host.inl.
#pragma once
#include "../../include/sph.h"
#include "sph_kernels.cuh"

namespace sphk {

__device__ __forceinline__ float dot3_rn(float a0, float a1, float a2, float b0, float b1, float b2) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

// The isometry of a posed shape, world = rot * local + t (row-major rotation), and the rigid motion of the body behind it.
struct Pose {
    float rot[9], t[3];
};
struct BodyVel {
    float linvel[3], angvel[3], com[3];
    int moving;  // 0: no parent body, velocity 0 (fluids_pipeline.rs:184-186)
};
// local = rot^T (world - t), every operation an explicit round-to-nearest one
__device__ __forceinline__ void to_local_rn(const Pose& P, float wx, float wy, float wz, float* l) {
    const float dx = __fsub_rn(wx, P.t[0]), dy = __fsub_rn(wy, P.t[1]), dz = __fsub_rn(wz, P.t[2]);
    l[0] = dot3_rn(P.rot[0], P.rot[3], P.rot[6], dx, dy, dz);
    l[1] = dot3_rn(P.rot[1], P.rot[4], P.rot[7], dx, dy, dz);
    l[2] = dot3_rn(P.rot[2], P.rot[5], P.rot[8], dx, dy, dz);
}
// body.velocity_at_point(x) = linvel + angvel x (x - world_com), likewise
__device__ __forceinline__ void body_velocity_at(const BodyVel& b, float x, float y, float z, float* v) {
    const float dx = __fsub_rn(x, b.com[0]), dy = __fsub_rn(y, b.com[1]), dz = __fsub_rn(z, b.com[2]);
    v[0] = __fadd_rn(b.linvel[0], __fsub_rn(__fmul_rn(b.angvel[1], dz), __fmul_rn(b.angvel[2], dy)));
    v[1] = __fadd_rn(b.linvel[1], __fsub_rn(__fmul_rn(b.angvel[2], dx), __fmul_rn(b.angvel[0], dz)));
    v[2] = __fadd_rn(b.linvel[2], __fsub_rn(__fmul_rn(b.angvel[0], dy), __fmul_rn(b.angvel[1], dx)));
}

// ---- parry HeightField (DESIGN.md section 11 geometry), shared by the sampler and the point query ----------------------
// cell index and fraction of coordinate c on a grid of `cells` cells of size d starting at -half
__device__ __forceinline__ int smp_cell(float c, float half, float d, int cells, float* frac) {
    const float t = __fdiv_rn(__fadd_rn(c, half), d);
    const int i = min(max((int)floorf(t), 0), cells - 1);
    *frac = __fsub_rn(t, (float)i);
    return i;
}

__device__ __forceinline__ float smp_grid(int j, int last, float half, float d) {
    return j == last ? half : __fadd_rn(-half, __fmul_rn((float)j, d));
}

struct HfGrid {
    const float* hgt;         // nrows * ncols heights, row-major: rows along z, columns along x
    int nrows, ncols;
    float hx, hz, dx, dz, sy; // half extents in x and z, cell sizes, height scale
    float dmin;               // min(dx, dz)
    float cap2, margin;       // the search's cap (squared) and its margin M (DESIGN.md section 10)
};

// Closest point q of the closed triangle (a, b, c) to p and its squared distance: Ericson, Real-Time Collision Detection
// 5.1.5 (vertex, edge and face regions), every operation an explicit round-to-nearest one.
__device__ __forceinline__ float hf_tri(const float* p, const float* a, const float* b, const float* c, float* q) {
    const float ab[3] = {__fsub_rn(b[0], a[0]), __fsub_rn(b[1], a[1]), __fsub_rn(b[2], a[2])};
    const float ac[3] = {__fsub_rn(c[0], a[0]), __fsub_rn(c[1], a[1]), __fsub_rn(c[2], a[2])};
    const float ap[3] = {__fsub_rn(p[0], a[0]), __fsub_rn(p[1], a[1]), __fsub_rn(p[2], a[2])};
    const float d1 = dot3_rn(ab[0], ab[1], ab[2], ap[0], ap[1], ap[2]), d2 = dot3_rn(ac[0], ac[1], ac[2], ap[0], ap[1], ap[2]);
    const float bp[3] = {__fsub_rn(p[0], b[0]), __fsub_rn(p[1], b[1]), __fsub_rn(p[2], b[2])};
    const float d3 = dot3_rn(ab[0], ab[1], ab[2], bp[0], bp[1], bp[2]), d4 = dot3_rn(ac[0], ac[1], ac[2], bp[0], bp[1], bp[2]);
    const float cp[3] = {__fsub_rn(p[0], c[0]), __fsub_rn(p[1], c[1]), __fsub_rn(p[2], c[2])};
    const float d5 = dot3_rn(ab[0], ab[1], ab[2], cp[0], cp[1], cp[2]), d6 = dot3_rn(ac[0], ac[1], ac[2], cp[0], cp[1], cp[2]);
    const float vc = __fsub_rn(__fmul_rn(d1, d4), __fmul_rn(d3, d2));
    const float vb = __fsub_rn(__fmul_rn(d5, d2), __fmul_rn(d1, d6));
    const float va = __fsub_rn(__fmul_rn(d3, d6), __fmul_rn(d5, d4));
    const float e43 = __fsub_rn(d4, d3), e56 = __fsub_rn(d5, d6);
    if (d1 <= 0.f && d2 <= 0.f) {
        q[0] = a[0]; q[1] = a[1]; q[2] = a[2];
    } else if (d3 >= 0.f && d4 <= d3) {
        q[0] = b[0]; q[1] = b[1]; q[2] = b[2];
    } else if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
        const float v = __fdiv_rn(d1, __fsub_rn(d1, d3));
        for (int k = 0; k < 3; ++k) q[k] = __fadd_rn(a[k], __fmul_rn(v, ab[k]));
    } else if (d6 >= 0.f && d5 <= d6) {
        q[0] = c[0]; q[1] = c[1]; q[2] = c[2];
    } else if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
        const float v = __fdiv_rn(d2, __fsub_rn(d2, d6));
        for (int k = 0; k < 3; ++k) q[k] = __fadd_rn(a[k], __fmul_rn(v, ac[k]));
    } else if (va <= 0.f && e43 >= 0.f && e56 >= 0.f) {
        const float v = __fdiv_rn(e43, __fadd_rn(e43, e56));
        for (int k = 0; k < 3; ++k) q[k] = __fadd_rn(b[k], __fmul_rn(v, __fsub_rn(c[k], b[k])));
    } else {
        const float den = __fdiv_rn(1.f, __fadd_rn(__fadd_rn(va, vb), vc));
        const float v = __fmul_rn(vb, den), w = __fmul_rn(vc, den);
        for (int k = 0; k < 3; ++k) q[k] = __fadd_rn(__fadd_rn(a[k], __fmul_rn(ab[k], v)), __fmul_rn(ac[k], w));
    }
    const float e[3] = {__fsub_rn(p[0], q[0]), __fsub_rn(p[1], q[1]), __fsub_rn(p[2], q[2])};
    return dot3_rn(e[0], e[1], e[2], e[0], e[1], e[2]);
}

// Both triangles of cell (i, j), (p00, p10, p01) and (p10, p11, p01), into the running best: the lexicographic minimum of
// (squared distance, parry triangle index 2 (j (nrows - 1) + i) + t), so the visit order cannot change a tie.
__device__ __forceinline__ void hf_cell(const HfGrid& g, int i, int j, const float* p, float& best, uint32_t& bidx, float* q) {
    const int ni = g.nrows - 1, nj = g.ncols - 1;
    const float x0 = smp_grid(j, nj, g.hx, g.dx), x1 = smp_grid(j + 1, nj, g.hx, g.dx);
    const float z0 = smp_grid(i, ni, g.hz, g.dz), z1 = smp_grid(i + 1, ni, g.hz, g.dz);
    const float* r0 = g.hgt + (size_t)i * g.ncols + j;
    const float p00[3] = {x0, __fmul_rn(__ldg(r0), g.sy), z0};
    const float p10[3] = {x1, __fmul_rn(__ldg(r0 + 1), g.sy), z0};
    const float p01[3] = {x0, __fmul_rn(__ldg(r0 + g.ncols), g.sy), z1};
    const float p11[3] = {x1, __fmul_rn(__ldg(r0 + g.ncols + 1), g.sy), z1};
    const uint32_t base = 2u * ((uint32_t)j * (uint32_t)ni + (uint32_t)i);
    float t[3];
    float d = hf_tri(p, p00, p10, p01, t);
    if (d < best || (d == best && base < bidx)) { best = d; bidx = base; q[0] = t[0]; q[1] = t[1]; q[2] = t[2]; }
    d = hf_tri(p, p10, p11, p01, t);
    if (d < best || (d == best && base + 1u < bidx)) { best = d; bidx = base + 1u; q[0] = t[0]; q[1] = t[1]; q[2] = t[2]; }
}

// HeightField::project_local_point (parry query/point/point_heightfield.rs): the closest point q over all triangles of a
// local point, is_inside always false.  Cells are searched in square rings around the point's (x, z) cell, clipped to the
// field; ring r lies at least (r - 1) dmin away horizontally, and the search stops once (r - 1) dmin - M exceeds both the
// best distance and the cap.  M covers the float32 error of every distance, so a triangle within the cap is never missed
// and the result equals the all-triangle minimum wherever it lies within the cap.  *d2 = |p - q|^2; false: no triangle.
__device__ __forceinline__ bool hf_closest(const HfGrid& g, float lx, float ly, float lz, float* q, float* d2) {
    const float p[3] = {lx, ly, lz};
    const int ni = g.nrows - 1, nj = g.ncols - 1;
    float fu, fv;
    const int ci = smp_cell(lz, g.hz, g.dz, ni, &fv), cj = smp_cell(lx, g.hx, g.dx, nj, &fu);
    const int rmax = max(max(ci, ni - 1 - ci), max(cj, nj - 1 - cj));
    float best = __int_as_float(0x7f800000);
    uint32_t bidx = UINT32_MAX;
    for (int r = 0; r <= rmax; ++r) {
        const float gap = __fsub_rn(__fmul_rn((float)(r - 1), g.dmin), g.margin);
        if (gap > 0.f && __fmul_rn(gap, gap) > fminf(best, g.cap2)) break;
        const int i0 = max(ci - r, 0), i1 = min(ci + r, ni - 1);
        for (int i = i0; i <= i1; ++i) {
            if (i == ci - r || i == ci + r) {
                const int j1 = min(cj + r, nj - 1);
                for (int j = max(cj - r, 0); j <= j1; ++j) hf_cell(g, i, j, p, best, bidx, q);
            } else {
                if (cj - r >= 0) hf_cell(g, i, cj - r, p, best, bidx, q);
                if (cj + r < nj) hf_cell(g, i, cj + r, p, best, bidx, q);
            }
        }
    }
    *d2 = best;
    return bidx != UINT32_MAX;
}

// Solids of revolution about local y: SPH_SHAPE_CYLINDER and SPH_SHAPE_CONE, a = half height, r = (base) radius; the cone's apex is
// at (0, a, 0) and its base disc at y = -a.  Every query is a 2-D one in the meridian half-plane (rho, y), rho = |(x, z)|,
// on the closed section [0, r] x [-a, a] or the triangle (0, a), (r, -a), (0, -a).  Outside: the closest point of the
// section.  Inside, surface included: the foot on the nearest surface edge (the axis is no surface); a tie goes to the side
// (the cone's slant), then to the bottom (base), then to the top.  keep: the foot keeps the point's rho.
__device__ __forceinline__ void rev_meridian(int kind, float a, float r, float rho, float y, float& qr, float& qy, bool& inside, bool& keep) {
    if (kind == SPH_SHAPE_CYLINDER) {
        inside = rho <= r && fabsf(y) <= a;
        if (inside) {
            const float ds = __fsub_rn(r, rho), db = __fadd_rn(y, a), dt = __fsub_rn(a, y);
            keep = !(ds <= db && ds <= dt);
            qr = keep ? rho : r;
            qy = !keep ? y : db <= dt ? -a : a;
        } else {
            keep = rho <= r;
            qr = keep ? rho : r;
            qy = fminf(fmaxf(y, -a), a);
        }
        return;
    }
    const float a2 = __fadd_rn(a, a);
    const float L2 = __fadd_rn(__fmul_rn(r, r), __fmul_rn(a2, a2));
    const float num = __fsub_rn(__fmul_rn(r, __fsub_rn(a, y)), __fmul_rn(a2, rho));  // |slant| times the depth below the slant
    inside = y >= -a && y <= a && rho <= r && num >= 0.f;
    if (inside) {
        keep = !(L2 > 0.f && __fdiv_rn(num, __fsqrt_rn(L2)) <= __fadd_rn(y, a));
        if (!keep) {  // the foot on the slant: the point plus depth times the unit normal (2a, r) / |slant|
            const float w = __fdiv_rn(num, L2);
            qr = __fadd_rn(rho, __fmul_rn(w, a2));
            qy = __fadd_rn(y, __fmul_rn(w, r));
        } else {
            qr = rho;
            qy = -a;
        }
    } else if (y < -a && rho <= r) {  // under the base disc
        keep = true;
        qr = rho;
        qy = -a;
    } else {  // the slant from the apex (0, a) to the rim (r, -a), its parameter clamped to the segment
        keep = false;
        const float s = L2 > 0.f ? fminf(fmaxf(__fdiv_rn(__fadd_rn(__fmul_rn(r, rho), __fmul_rn(a2, __fsub_rn(a, y))), L2), 0.f), 1.f) : 0.f;
        qr = __fmul_rn(s, r);
        qy = __fsub_rn(a, __fmul_rn(s, a2));
    }
}
__host__ __device__ __forceinline__ bool is_rev(int kind) { return kind == SPH_SHAPE_CYLINDER || kind == SPH_SHAPE_CONE; }
__device__ __forceinline__ float rev_rho(float lx, float lz) { return __fsqrt_rn(__fadd_rn(__fmul_rn(lx, lx), __fmul_rn(lz, lz))); }

// LiquidWorld::particles_intersecting_aabb liquid_world.rs:211-243 over HGrid::cells_intersecting_aabb hgrid.rs:122-133.
// One thread per cell of the (clipped) cell box [key(mins), key(maxs)] of the grid built by the last step; the CURRENT
// positions are tested (Aabb::distance_to_point, solid: norm of the per-axis excess) against particle_radius.
// out[2k] = kind (0 fluid, 1 boundary), out[2k+1] = original index; order is whatever the atomics give (host sorts).
struct AabbQuery {
    int lx, ly, lz, dx, dy, dz;  // first cell and extent (cells) of the box
    float mins[3], maxs[3], radius;
    uint32_t slot_lo, slot_hi;   // owned fluid slots (ghost copies of a slab world are skipped)
    // particles_intersecting_shape (liquid_world.rs:246-281): kind 0 = the box itself (distance < radius, :224), else the
    // SPH_SHAPE_* kind (the capsule's segment along local y), posed by the isometry `pose`: point p is hit when
    // shape.distance_to_point(pos, p, solid) <= radius (:263)
    int kind;
    Pose pose;
    float sp[3];                 // ball: radius; cuboid: half extents; capsule, cylinder, cone: half height, radius
    HfGrid hf;                   // SPH_SHAPE_HEIGHTFIELD (k_aabb_query<true>): cap = radius
};
// HF: the heightfield only; REV: cylinder and cone only (k_aabb_query<false, true>); neither: the box, ball, cuboid, capsule.
template <bool HF, bool REV = false>
__device__ __forceinline__ bool query_near(const AabbQuery& q, const float4& p) {
    if (REV) {  // distance_to_point(solid): 0 inside, else the meridian distance to the closest point of the section
        float l[3];
        to_local_rn(q.pose, p.x, p.y, p.z, l);
        const float rho = rev_rho(l[0], l[2]);
        float qr, qy;
        bool in, keep;
        rev_meridian(q.kind, q.sp[0], q.sp[1], rho, l[1], qr, qy, in, keep);
        if (in) return true;
        const float dr = __fsub_rn(rho, qr), dy = __fsub_rn(l[1], qy);
        return __fsqrt_rn(__fadd_rn(__fmul_rn(dr, dr), __fmul_rn(dy, dy))) <= q.radius;
    }
    if (!HF && q.kind == 0) {
        float ex = fmaxf(fmaxf(q.mins[0] - p.x, p.x - q.maxs[0]), 0.f);
        float ey = fmaxf(fmaxf(q.mins[1] - p.y, p.y - q.maxs[1]), 0.f);
        float ez = fmaxf(fmaxf(q.mins[2] - p.z, p.z - q.maxs[2]), 0.f);
        return __fsqrt_rn(dist2_exact(ex, ey, ez)) < q.radius;
    }
    // local point = rot^T (p - t), in plain operations the compiler may contract: not to_local_rn, whose different rounding
    // would move points across the `<= radius` edge
    const float* rot = q.pose.rot;
    const float wx = p.x - q.pose.t[0], wy = p.y - q.pose.t[1], wz = p.z - q.pose.t[2];
    const float lx = rot[0] * wx + rot[3] * wy + rot[6] * wz;
    const float ly = rot[1] * wx + rot[4] * wy + rot[7] * wz;
    const float lz = rot[2] * wx + rot[5] * wy + rot[8] * wz;
    float d;
    if (HF) {  // HeightField::distance_to_point: the unsigned distance to the closest point (is_inside is always false)
        float c[3], d2;
        return hf_closest(q.hf, lx, ly, lz, c, &d2) && __fsqrt_rn(d2) <= q.radius;
    } else if (q.kind == SPH_SHAPE_BALL) {
        d = fmaxf(__fsqrt_rn(dist2_exact(lx, ly, lz)) - q.sp[0], 0.f);
    } else if (q.kind == SPH_SHAPE_CUBOID) {
        float ex = fmaxf(fabsf(lx) - q.sp[0], 0.f), ey = fmaxf(fabsf(ly) - q.sp[1], 0.f), ez = fmaxf(fabsf(lz) - q.sp[2], 0.f);
        d = __fsqrt_rn(dist2_exact(ex, ey, ez));
    } else {
        float cy = fminf(fmaxf(ly, -q.sp[0]), q.sp[0]);  // closest point of the segment
        d = fmaxf(__fsqrt_rn(dist2_exact(lx, ly - cy, lz)) - q.sp[1], 0.f);
    }
    return d <= q.radius;
}
// ColliderCouplingManager::update_boundaries, StaticSampling (fluids_pipeline.rs:180-191): the coupled boundary's particles
// are the collider's local sample points under its pose, world = rot * local + t, with the
// body's velocity_at_point(pt) = linvel + angvel x (pt - world_com) evaluated at the LOCAL point, as :183 does.  Explicit
// round-to-nearest operations (no contraction into FMAs) keep the result a fixed float32 expression a host can restate.
struct ColliderPose {
    Pose pose;
    BodyVel body;
};
// One thread per SORTED boundary slot; the slots whose original index lies in [first, first + n) belong to the collider.
__global__ void k_collider_static(uint32_t nb, const uint32_t* __restrict__ borig, uint32_t first, uint32_t n, const float4* __restrict__ local,
                                  ColliderPose P, float4* __restrict__ bpos, float4* __restrict__ bvel) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nb) return;
    const uint32_t k = borig[s] - first;
    if (k >= n) return;
    const float4 l = local[k];
    const float* rot = P.pose.rot;
    bpos[s] = make_float4(__fadd_rn(dot3_rn(rot[0], rot[1], rot[2], l.x, l.y, l.z), P.pose.t[0]),
                          __fadd_rn(dot3_rn(rot[3], rot[4], rot[5], l.x, l.y, l.z), P.pose.t[1]),
                          __fadd_rn(dot3_rn(rot[6], rot[7], rot[8], l.x, l.y, l.z), P.pose.t[2]), 0.f);
    float v[3] = {0.f, 0.f, 0.f};
    if (P.body.moving) body_velocity_at(P.body, l.x, l.y, l.z, v);
    bvel[s] = make_float4(v[0], v[1], v[2], bvel[s].w);  // .w carries the boundary slot
}
// transmit_forces (fluids_pipeline.rs:263-287): the impulse body.apply_impulse_at_point(force * dt, pos) gives the body,
// summed over the collider's boundary particles: out[6k..] = (sum f dt, sum (p - com) x f dt) of collider slot k.  One
// launch for all colliders, each boundary slot read once: a block sums its slots per collider in shared memory and adds
// the non-zero sums to `out` (zeroed before).  The float atomics make the last bits depend on timing.
struct ImpulseTable {
    int collider[MAX_BOUNDARIES];   // boundary slot -> collider slot whose impulse it feeds, or -1
    float com[MAX_BOUNDARIES][3];   // per collider slot: the body's world centre of mass
};
__global__ void k_collider_impulse(uint32_t nb, const float4* __restrict__ bpos, const float4* __restrict__ bvel, const float* __restrict__ bforce,
                                   float dt, ImpulseTable T, float* __restrict__ out) {
    __shared__ float acc[MAX_BOUNDARIES][6];
    for (int k = threadIdx.x; k < MAX_BOUNDARIES * 6; k += blockDim.x) (&acc[0][0])[k] = 0.f;
    __syncthreads();
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < nb; s += gridDim.x * blockDim.x) {
        const int k = T.collider[fid_of(bvel[s])];
        if (k < 0) continue;
        const float fx = bforce[3 * (size_t)s] * dt, fy = bforce[3 * (size_t)s + 1] * dt, fz = bforce[3 * (size_t)s + 2] * dt;
        const float4 p = bpos[s];
        const float rx = p.x - T.com[k][0], ry = p.y - T.com[k][1], rz = p.z - T.com[k][2];
        atomicAdd(&acc[k][0], fx);
        atomicAdd(&acc[k][1], fy);
        atomicAdd(&acc[k][2], fz);
        atomicAdd(&acc[k][3], ry * fz - rz * fy);
        atomicAdd(&acc[k][4], rz * fx - rx * fz);
        atomicAdd(&acc[k][5], rx * fy - ry * fx);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < MAX_BOUNDARIES * 6; k += blockDim.x) {
        const float v = (&acc[0][0])[k];
        if (v != 0.f) atomicAdd(&out[k], v);
    }
}

// ColliderCouplingManager::update_boundaries, DynamicContactSampling (fluids_pipeline.rs:192-255).  Each candidate fluid
// particle is handled by one thread, which runs every contact collider whose cell box holds the particle's cell (of its
// position at the start of the substep), in collider-slot order: a particle's pushes depend only on its own state and on
// earlier colliders, so this is the reference's collider-major loop with slot order standing in for hash-map order.  The
// pass does not write the fluid: it appends sample and push records (k_contact_apply writes the pushes), so it can be
// re-run with larger buffers when they overflow.  Every operation is an explicit round-to-nearest one, a fixed float32
// expression a host can restate.
struct ContactCollider {
    int kind;                       // SPH_SHAPE_*: ball (sp[0] radius), cuboid (sp half extents), heightfield; capsule, cylinder, cone
                                    // along local y (sp[0] half height, sp[1] radius)
    uint32_t slot;                  // collider slot: the samples' sort key
    Pose pose;
    float sp[3];
    float mins[3], maxs[3];         // the posed shape's AABB loosened by h + prediction
    int clo[3], chi[3];             // its cell box [key(mins), key(maxs)]
    BodyVel body;                   // not moving: sample velocity 0
    uint32_t first_bin;             // first enumeration index of this collider's (grid-clipped) bin box
    int bl[3], bd[3];               // that bin box: first bin and extent per axis
};
struct ContactResults {                     // what contact sampling reduces, read back with one copy
    uint32_t samples, pushes;                  // records k_contact_sample made (past the capacities too: the pass is re-run)
    CellBox fluid, bound;                      // the cell boxes of the fluid after the pushes and of the rebuilt boundaries
    uint32_t per_collider[MAX_BOUNDARIES];     // samples per collider slot
};
struct ContactParams {
    const ContactCollider* col;
    int nc;                         // contact colliders, ascending slot
    uint32_t total_bins;
    float dt, cut, margin;          // lagging dt, h + prediction, 0.1 particle_radius
    uint32_t cap_s, cap_p;
    const HfGrid* hf;               // k_contact_sample<true>: per collider (same index as col), the grid of a heightfield
};
__device__ __forceinline__ bool contact_in_box(const ContactCollider& c, int cx, int cy, int cz) {
    return cx >= c.clo[0] && cx <= c.chi[0] && cy >= c.clo[1] && cy <= c.chi[1] && cz >= c.clo[2] && cz <= c.chi[2];
}
// project_point_and_get_feature, non-solid, in the shape's local frame: false when the projection is undefined (ball centre)
template <bool REV>
__device__ __forceinline__ bool contact_project_local(const ContactCollider& c, float lx, float ly, float lz, float* q, bool* inside) {
    if (REV && is_rev(c.kind)) {  // the meridian foot lifted along u = (x, z) / rho, along local +x at rho = 0
        const float rho = rev_rho(lx, lz);
        float qr, qy;
        bool keep;
        rev_meridian(c.kind, c.sp[0], c.sp[1], rho, ly, qr, qy, *inside, keep);
        if (keep) {
            q[0] = lx; q[2] = lz;
        } else if (rho == 0.f) {
            q[0] = qr; q[2] = 0.f;
        } else {
            const float s = __fdiv_rn(qr, rho);
            q[0] = __fmul_rn(lx, s); q[2] = __fmul_rn(lz, s);
        }
        q[1] = qy;
    } else if (c.kind == SPH_SHAPE_BALL) {  // parry Ball::project_local_point
        const float n2 = dot3_rn(lx, ly, lz, lx, ly, lz);
        if (n2 == 0.f) return false;  // parry divides by zero here (NaN): no sample, no push
        *inside = n2 <= __fmul_rn(c.sp[0], c.sp[0]);
        const float s = __fdiv_rn(c.sp[0], __fsqrt_rn(n2));
        q[0] = __fmul_rn(lx, s); q[1] = __fmul_rn(ly, s); q[2] = __fmul_rn(lz, s);
    } else if (c.kind == SPH_SHAPE_CUBOID) {  // parry Aabb::project_local_point over [-e, e]
        const float l[3] = {lx, ly, lz};
        float mp[3], pm[3], sh[3];
        bool in = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            mp[a] = __fsub_rn(-c.sp[a], l[a]);
            pm[a] = __fsub_rn(l[a], c.sp[a]);
            sh[a] = __fsub_rn(fmaxf(mp[a], 0.f), fmaxf(pm[a], 0.f));
            in = in && sh[a] == 0.f;
        }
        if (in) {  // nearest face; a tie goes to the mins face, a tie across axes keeps the lowest axis
            float best = -3.402823466e38f;
            int id = 0;
            bool is_mins = false;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                if (mp[a] < pm[a]) {
                    if (pm[a] > best) { id = a; is_mins = false; best = pm[a]; }
                } else if (mp[a] > best) { id = a; is_mins = true; best = mp[a]; }
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) sh[a] = a == id ? (is_mins ? best : -best) : 0.f;
        }
        *inside = in;
#pragma unroll
        for (int a = 0; a < 3; ++a) q[a] = __fadd_rn(l[a], sh[a]);
    } else {  // capsule: closest segment point, then out along (l - c) by the radius; on the axis along local +x
        const float cy = fminf(fmaxf(ly, -c.sp[0]), c.sp[0]);
        const float dy = __fsub_rn(ly, cy);
        const float dn = __fsqrt_rn(dot3_rn(lx, dy, lz, lx, dy, lz));
        *inside = dn <= c.sp[1];
        if (dn == 0.f) {
            q[0] = c.sp[1]; q[1] = cy; q[2] = 0.f;
        } else {
            const float s = __fdiv_rn(c.sp[1], dn);
            q[0] = __fmul_rn(lx, s); q[1] = __fadd_rn(cy, __fmul_rn(dy, s)); q[2] = __fmul_rn(lz, s);
        }
    }
    return true;
}
// One warp per enumerated bin (the bins of each collider's cell box, clipped to the grid); its lanes take the bin's particles.
// A particle is processed by the enumeration of the lowest-slot collider whose box holds its cell.  Records:
// samples  s4[2r] = (proj, orig), s4[2r+1] = (velocity, 0), key[r] = slot << 32 | orig, val[r] = r;
// pushes   p4[2r] = (new position, sorted slot), p4[2r+1] = (new velocity, 0).
// HF: the instantiations for worlds with a heightfield collider, REV: with a cylinder or cone collider; a world with
// neither runs k_contact_sample<false, false>, without their code.
template <bool HF, bool REV>
__global__ void k_contact_sample(ContactParams P, const float4* __restrict__ pos, const float4* __restrict__ vel, const uint32_t* __restrict__ cstart,
                                 const uint32_t* __restrict__ orig, float4* __restrict__ s4, unsigned long long* __restrict__ key, uint32_t* __restrict__ val,
                                 float4* __restrict__ p4, ContactResults* __restrict__ res) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= P.total_bins) return;  // warp-uniform
    int e = 0;
    while (e + 1 < P.nc && P.col[e + 1].first_bin <= warp) ++e;
    const ContactCollider& E = P.col[e];
    const uint32_t t = warp - E.first_bin;
    const int bz = E.bl[2] + (int)(t % (uint32_t)E.bd[2]);
    const int by = E.bl[1] + (int)((t / (uint32_t)E.bd[2]) % (uint32_t)E.bd[1]);
    const int bx = E.bl[0] + (int)(t / (uint32_t)(E.bd[2] * E.bd[1]));
    const int cell = cell_id(bx, by, bz);
    const uint32_t start = cstart[cell], end = cstart[cell + 1];
    CellBox box = CELL_BOX_EMPTY;
    for (uint32_t base = start; base < end; base += 32) {
        const uint32_t j = base + lane;
        bool mine = j < end;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f), v = p;
        int cx = 0, cy = 0, cz = 0;
        if (mine) {
            p = pos[j];
            v = vel[j];
            cx = cell_coord(p.x); cy = cell_coord(p.y); cz = cell_coord(p.z);
            mine = contact_in_box(E, cx, cy, cz);
            for (int k = 0; k < e && mine; ++k) mine = !contact_in_box(P.col[k], cx, cy, cz);
        }
        bool pushed = false;
        for (int k = e; k < P.nc; ++k) {  // warp-uniform loop: every lane reaches the ballots
            const ContactCollider& K = P.col[k];
            bool emit = false;
            float q[3] = {0.f, 0.f, 0.f}, sv[3] = {0.f, 0.f, 0.f};
            if (mine && contact_in_box(K, cx, cy, cz)) {
                const float pr[3] = {__fadd_rn(p.x, __fmul_rn(v.x, P.dt)), __fadd_rn(p.y, __fmul_rn(v.y, P.dt)), __fadd_rn(p.z, __fmul_rn(v.z, P.dt))};
                emit = pr[0] >= K.mins[0] && pr[0] <= K.maxs[0] && pr[1] >= K.mins[1] && pr[1] <= K.maxs[1] && pr[2] >= K.mins[2] &&
                       pr[2] <= K.maxs[2];
                float lq[3];
                bool inside = false;
                if (emit) {
                    float l[3];
                    to_local_rn(K.pose, pr[0], pr[1], pr[2], l);
                    if (HF && K.kind == SPH_SHAPE_HEIGHTFIELD) {  // a heightfield never has the point inside: samples only, no push
                        float d2;
                        emit = hf_closest(P.hf[k], l[0], l[1], l[2], lq, &d2);
                    } else {
                        emit = contact_project_local<REV>(K, l[0], l[1], l[2], lq, &inside);
                    }
                }
                if (emit) {
#pragma unroll
                    for (int a = 0; a < 3; ++a)
                        q[a] = __fadd_rn(dot3_rn(K.pose.rot[3 * a], K.pose.rot[3 * a + 1], K.pose.rot[3 * a + 2], lq[0], lq[1], lq[2]), K.pose.t[a]);
                    const float d[3] = {__fsub_rn(pr[0], q[0]), __fsub_rn(pr[1], q[1]), __fsub_rn(pr[2], q[2])};
                    const float depth = __fsqrt_rn(dot3_rn(d[0], d[1], d[2], d[0], d[1], d[2]));
                    if (depth > F32_EPS) {  // Unit::try_new_and_get(dpt, f32::EPSILON)
                        const float n[3] = {__fdiv_rn(d[0], depth), __fdiv_rn(d[1], depth), __fdiv_rn(d[2], depth)};
                        if (inside) {
                            const float s = __fadd_rn(depth, P.margin);
                            p.x = __fsub_rn(p.x, __fmul_rn(n[0], s));
                            p.y = __fsub_rn(p.y, __fmul_rn(n[1], s));
                            p.z = __fsub_rn(p.z, __fmul_rn(n[2], s));
                            const float ve = dot3_rn(n[0], n[1], n[2], v.x, v.y, v.z);
                            if (ve > 0.f) {
                                v.x = __fsub_rn(v.x, __fmul_rn(n[0], ve));
                                v.y = __fsub_rn(v.y, __fmul_rn(n[1], ve));
                                v.z = __fsub_rn(v.z, __fmul_rn(n[2], ve));
                            }
                            pushed = true;
                        } else if (depth > P.cut) {
                            emit = false;
                        }
                    }
                }
                if (emit && K.body.moving) body_velocity_at(K.body, q[0], q[1], q[2], sv);  // at the WORLD point
            }
            const unsigned m = __ballot_sync(0xffffffffu, emit);
            if (!m) continue;
            uint32_t r0 = 0;
            if (lane == 0) {
                r0 = atomicAdd(&res->samples, (uint32_t)__popc(m));
                atomicAdd(&res->per_collider[K.slot], (uint32_t)__popc(m));
            }
            r0 = __shfl_sync(0xffffffffu, r0, 0);
            if (emit) {
                const uint32_t r = r0 + __popc(m & ((1u << lane) - 1u));
                const uint32_t o = orig[j];
                cell_box_add(box, q[0], q[1], q[2], C.h);
                if (r < P.cap_s) {
                    s4[2 * (size_t)r] = make_float4(q[0], q[1], q[2], __uint_as_float(o));
                    s4[2 * (size_t)r + 1] = make_float4(sv[0], sv[1], sv[2], 0.f);
                    key[r] = (unsigned long long)K.slot << 32 | o;
                    val[r] = r;
                }
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, pushed);
        if (m) {
            uint32_t r0 = 0;
            if (lane == 0) r0 = atomicAdd(&res->pushes, (uint32_t)__popc(m));
            r0 = __shfl_sync(0xffffffffu, r0, 0);
            const uint32_t r = r0 + __popc(m & ((1u << lane) - 1u));
            if (pushed && r < P.cap_p) {
                p4[2 * (size_t)r] = make_float4(p.x, p.y, p.z, __uint_as_float(j));
                p4[2 * (size_t)r + 1] = make_float4(v.x, v.y, v.z, 0.f);
            }
        }
    }
    cell_box_commit_warp(box, &res->bound);
}
// The pushes of k_contact_sample, written only when neither record buffer overflowed (the pass is then re-run unchanged).
__global__ void k_contact_apply(const float4* __restrict__ p4, const ContactResults* __restrict__ res, uint32_t cap_s, uint32_t cap_p, float4* __restrict__ pos,
                                float4* __restrict__ vel) {
    const uint32_t ns = res->samples, np = res->pushes;
    if (ns > cap_s || np > cap_p) return;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < np; r += gridDim.x * blockDim.x) {
        const float4 a = p4[2 * (size_t)r], b = p4[2 * (size_t)r + 1];
        const uint32_t s = __float_as_uint(a.w);
        pos[s] = make_float4(a.x, a.y, a.z, pos[s].w);
        vel[s] = make_float4(b.x, b.y, b.z, vel[s].w);
    }
}
// Cell bounds of the boundary particles that stay (boundaries not coupled by contact sampling: skip bit set).
__global__ void k_bounds_kept(const float4* __restrict__ bpos, const float4* __restrict__ bvel, uint32_t n, unsigned long long skip, CellBox* __restrict__ out) {
    CellBox box = CELL_BOX_EMPTY;
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        if ((skip >> fid_of(bvel[s])) & 1ull) continue;
        const float4 p = bpos[s];
        cell_box_add(box, p.x, p.y, p.z, C.h);
    }
    cell_box_commit_warp(box, out);
}
// Rebuild of the boundary arrays in ORIGINAL order: the boundaries that stay move to their new offsets...
struct ContactRebuild {
    uint32_t old_off[MAX_BOUNDARIES], new_off[MAX_BOUNDARIES];
    unsigned long long skip;             // boundary slots refilled from samples
    uint32_t col_first[MAX_BOUNDARIES];  // per collider slot: its first record in the sorted samples
    uint32_t col_dst[MAX_BOUNDARIES];    // ... the new offset of its boundary
    uint32_t col_bslot[MAX_BOUNDARIES];  // ... and that boundary's slot
};
__global__ void k_contact_keep(uint32_t nb, const float4* __restrict__ bpos, const float4* __restrict__ bvel, const uint32_t* __restrict__ borig,
                               const ContactRebuild T, float4* __restrict__ opos, float4* __restrict__ ovel, uint32_t* __restrict__ oorig) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nb) return;
    const float4 v = bvel[s];
    const uint32_t b = fid_of(v);
    if ((T.skip >> b) & 1ull) return;
    const uint32_t d = T.new_off[b] + (borig[s] - T.old_off[b]);
    opos[d] = bpos[s];
    ovel[d] = v;
    oorig[d] = d;
}
// ... and the sorted samples (by collider slot, then original fluid index) fill the contact-coupled boundaries.
__global__ void k_contact_write(uint32_t n, const unsigned long long* __restrict__ key, const uint32_t* __restrict__ val, const float4* __restrict__ s4,
                                const ContactRebuild T, float4* __restrict__ opos, float4* __restrict__ ovel, uint32_t* __restrict__ oorig) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const uint32_t k = (uint32_t)(key[r] >> 32), src = val[r];
    const uint32_t d = T.col_dst[k] + (r - T.col_first[k]);
    const float4 a = s4[2 * (size_t)src], b = s4[2 * (size_t)src + 1];
    opos[d] = make_float4(a.x, a.y, a.z, 0.f);
    ovel[d] = make_float4(b.x, b.y, b.z, __uint_as_float(T.col_bslot[k]));
    oorig[d] = d;
}

template <bool HF, bool REV>
__global__ void k_aabb_query(AabbQuery q,const float4* __restrict__ pos, const uint32_t* __restrict__ cstart, const uint32_t* __restrict__ orig,
                             const float4* __restrict__ bpos, const uint32_t* __restrict__ bstart, const uint32_t* __restrict__ borig,
                             uint32_t* __restrict__ out, uint32_t cap, uint32_t* __restrict__ count) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint32_t)(q.dx * q.dy * q.dz)) return;
    int cz = q.lz + (int)(t % (uint32_t)q.dz);
    int cy = q.ly + (int)((t / (uint32_t)q.dz) % (uint32_t)q.dy);
    int cx = q.lx + (int)(t / (uint32_t)(q.dz * q.dy));
    int c = cell_id(cx, cy, cz);
    if (pos) {
        uint32_t s = max(cstart[c], q.slot_lo), e = min(cstart[c + 1], q.slot_hi);
        for (uint32_t j = s; j < e; ++j)
            if (query_near<HF, REV>(q, pos[j])) {
                uint32_t k = atomicAdd(count, 1u);
                if (k < cap) {
                    out[2 * (size_t)k] = 0u;
                    out[2 * (size_t)k + 1] = orig[j];
                }
            }
    }
    if (bpos) {
        for (uint32_t j = bstart[c]; j < bstart[c + 1]; ++j)
            if (query_near<HF, REV>(q, bpos[j])) {
                uint32_t k = atomicAdd(count, 1u);
                if (k < cap) {
                    out[2 * (size_t)k] = 1u;
                    out[2 * (size_t)k + 1] = borig[j];
                }
            }
    }
}

}  // namespace sphk
