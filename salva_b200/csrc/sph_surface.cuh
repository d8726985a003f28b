// sph_surface.cuh — fluid surface extraction (DESIGN.md section 15; host side in sph_surface_host.inl).
//
// The field phi(x) = sum_j V_j W(|x - x_j|) over the particles of the selected fluids is sampled on a lattice
// p_ijk = origin + spacing (i, j, k) and polygonised by marching tetrahedra on the Kuhn split of every lattice cube.  The
// particles are binned into cells of width h on the extractor's own scratch; the grid travels as a kernel argument, so
// nothing here reads or writes the step's grid constants (C.ox .. C.nz) or arrays.  C.h, C.inv_h and the kernel
// normalisations depend on h alone and are read as the step reads them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sphk {

struct SurfGrid {  // the extractor's cell grid: cells [o, o + n) of width h, z fastest
    int ox, oy, oz;
    int nx, ny, nz;
};
struct SurfLattice {
    float o[3];     // origin: spacing * floor(lo / spacing)
    float s;        // spacing
    uint32_t n[3];  // points per axis
    float iso;
};
struct SurfSel {  // which fluid slots are meshed, and where their particles go in the extractor's array
    uint32_t mask;
    uint32_t slot_off[MAX_FLUIDS];  // first original index of each fluid slot
    uint32_t out_off[MAX_FLUIDS];   // first row of the slot in the collected array
};

// The edge directions a lattice point owns, in vertex order: +x, +y, +z, +x+y, +x+z, +y+z, +x+y+z (bit a = axis a).
__constant__ uint8_t SURF_DIR_BITS[7] = {1, 2, 4, 3, 5, 6, 7};
// Kuhn tetrahedra (0, e_a, e_a + e_b, 1) in the order of the permutations (a, b, c): xyz, xzy, yxz, yzx, zxy, zyx; corner k's
// offset bits.  The odd permutations give negatively oriented tetrahedra, whose triangles are wound the other way.
__constant__ uint8_t SURF_TET[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
__constant__ uint8_t SURF_TET_ODD[6] = {0, 1, 1, 0, 0, 1};
// Tetrahedron edges (0,1) (0,2) (0,3) (1,2) (1,3) (2,3); their corners.
__constant__ uint8_t SURF_TET_EDGE[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
// Case table of a positively oriented tetrahedron: case = sum of 2^k over its inside corners k; per case the number of
// triangles and their edges, wound counter-clockwise seen from the outside (the side of lower phi).
__constant__ int8_t SURF_CASES[16][7] = {
    {0, 0, 0, 0, 0, 0, 0}, {1, 0, 1, 2, 0, 0, 0}, {1, 0, 4, 3, 0, 0, 0}, {2, 1, 2, 4, 1, 4, 3},
    {1, 1, 3, 5, 0, 0, 0}, {2, 0, 5, 2, 0, 3, 5}, {2, 0, 4, 5, 0, 5, 1}, {1, 2, 4, 5, 0, 0, 0},
    {1, 2, 5, 4, 0, 0, 0}, {2, 0, 1, 5, 0, 5, 4}, {2, 0, 5, 3, 0, 2, 5}, {1, 1, 5, 3, 0, 0, 0},
    {2, 1, 3, 4, 1, 4, 2}, {1, 0, 3, 4, 0, 0, 0}, {1, 0, 2, 1, 0, 0, 0}, {0, 0, 0, 0, 0, 0, 0}};

__device__ __forceinline__ int surf_dir_index(int bits) {  // inverse of SURF_DIR_BITS
    return bits == 1 ? 0 : bits == 2 ? 1 : bits == 4 ? 2 : bits == 3 ? 3 : bits == 5 ? 4 : bits == 6 ? 5 : 6;
}
// origin + (float)i * spacing, a round-to-nearest product and then a sum
__device__ __forceinline__ float surf_coord(const SurfLattice& L, int a, uint32_t i) { return __fadd_rn(L.o[a], __fmul_rn((float)i, L.s)); }

// float <-> unsigned keys whose unsigned order is the float order (AABB reductions with integer atomics)
__device__ __forceinline__ uint32_t surf_fkey(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// The selected fluids' particles of the device state, as (x, y, z, volume), the in-cell sort key (fluid slot, id) and, when
// vout is not null, the velocities (x, y, z, 0).
__global__ void k_surf_collect(uint32_t n, const float4* __restrict__ pos, const float4* __restrict__ vel, const uint32_t* __restrict__ orig,
                               const uint32_t* __restrict__ gid, SurfSel sel, const float* __restrict__ vol, float vol0, float4* __restrict__ out,
                               unsigned long long* __restrict__ key, float4* __restrict__ vout) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t f = fid_of(vel[i]);
    if (!((sel.mask >> f) & 1u)) return;
    const uint32_t g = orig[i];
    const uint32_t k = sel.out_off[f] + (g - sel.slot_off[f]);
    const float4 p = pos[i];
    out[k] = make_float4(p.x, p.y, p.z, vol ? vol[g] : vol0);
    key[k] = ((unsigned long long)f << 32) | gid[i];
    if (vout) {
        const float4 v = vel[i];
        vout[k] = make_float4(v.x, v.y, v.z, 0.f);
    }
}

// AABB of the finite positions: out[0..2] min keys, out[3..5] max keys (surf_fkey)
__global__ void k_surf_aabb(uint32_t n, const float4* __restrict__ p4, uint32_t* __restrict__ out) {
    uint32_t mn[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, mx[3] = {0u, 0u, 0u};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = p4[i];
        const float c[3] = {p.x, p.y, p.z};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (!isfinite(c[a])) continue;
            mn[a] = min(mn[a], surf_fkey(c[a]));
            mx[a] = max(mx[a], surf_fkey(c[a]));
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&out[a], mn[a]);
            atomicMax(&out[3 + a], mx[a]);
        }
    }
}

// Counting sort into the extractor's cells; particles outside the grid (they reach no lattice point) get cid = ~0.
__global__ void k_surf_hist(uint32_t n, const float4* __restrict__ p4, SurfGrid g, uint32_t* __restrict__ cid, uint32_t* __restrict__ rank,
                            uint32_t* __restrict__ count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = p4[i];
    const float q[3] = {floorf(__fdiv_rn(p.x, C.h)), floorf(__fdiv_rn(p.y, C.h)), floorf(__fdiv_rn(p.z, C.h))};
    const int o[3] = {g.ox, g.oy, g.oz}, d[3] = {g.nx, g.ny, g.nz};
    int c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (!(q[a] >= (float)o[a] && q[a] < (float)o[a] + (float)d[a])) {  // NaN lands here too
            cid[i] = 0xFFFFFFFFu;
            return;
        }
        c[a] = (int)q[a] - o[a];
    }
    const uint32_t id = ((uint32_t)c[0] * (uint32_t)g.ny + (uint32_t)c[1]) * (uint32_t)g.nz + (uint32_t)c[2];
    cid[i] = id;
    rank[i] = atomicAdd(&count[id], 1u);
}

// Deterministic mode: each cell's slice of perm in ascending (fluid slot, id)
__global__ void k_surf_cell_sort(uint32_t ncell, const uint32_t* __restrict__ start, uint32_t* __restrict__ perm,
                                 const unsigned long long* __restrict__ key) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncell) return;
    const uint32_t s = start[c], e = start[c + 1];
    for (uint32_t a = s + 1; a < e; ++a) {
        const uint32_t v = perm[a];
        const unsigned long long kv = key[v];
        uint32_t b = a;
        while (b > s && key[perm[b - 1]] > kv) {
            perm[b] = perm[b - 1];
            --b;
        }
        perm[b] = v;
    }
}

// The particles of the 27 cells around x in a fixed order (x, then y, then the z-run of three cells): fn(j) for each
// sorted index j.  Returns false when every cell is empty.
template <class Fn>
__device__ __forceinline__ bool surf_for_cells(float x, float y, float z, const SurfGrid& g, const uint32_t* __restrict__ cstart, Fn&& fn) {
    const int cx = (int)floorf(__fdiv_rn(x, C.h)) - g.ox, cy = (int)floorf(__fdiv_rn(y, C.h)) - g.oy, cz = (int)floorf(__fdiv_rn(z, C.h)) - g.oz;
    const int z0 = max(cz - 1, 0), z1 = min(cz + 1, g.nz - 1);
    bool any = false;
    if (z0 > z1) return false;
    for (int ix = max(cx - 1, 0); ix <= min(cx + 1, g.nx - 1); ++ix)
        for (int iy = max(cy - 1, 0); iy <= min(cy + 1, g.ny - 1); ++iy) {
            const uint32_t base = ((uint32_t)ix * (uint32_t)g.ny + (uint32_t)iy) * (uint32_t)g.nz;
            const uint32_t s = cstart[base + z0], e = cstart[base + z1 + 1];
            any |= s < e;
            for (uint32_t j = s; j < e; ++j) fn(j);
        }
    return any;
}

// Sum over the particles of the 27 cells around x of V_j W(r) (G = false) or of V_j W'(r) / r (x - x_j) (G = true).
template <bool G>
__device__ __forceinline__ bool surf_gather(float x, float y, float z, const SurfGrid& g, const uint32_t* __restrict__ cstart,
                                            const float4* __restrict__ sp, float4& acc) {
    acc = make_float4(0.f, 0.f, 0.f, 0.f);
    return surf_for_cells(x, y, z, g, cstart, [&](uint32_t j) {
        const float4 pj = sp[j];
        const float dx = __fsub_rn(x, pj.x), dy = __fsub_rn(y, pj.y), dz = __fsub_rn(z, pj.z);
        const float d2 = dist2_exact(dx, dy, dz);
        if (!(d2 <= C.h2)) return;
        const float r = __fsqrt_rn(d2);
        if (G) {
            if (!(d2 > F32_EPS * F32_EPS)) return;
            const float gf = __fmul_rn(pj.w, __fdiv_rn(kernel_dw_kind(C.kg, r), r));
            acc.x = __fmaf_rn(gf, dx, acc.x);
            acc.y = __fmaf_rn(gf, dy, acc.y);
            acc.z = __fmaf_rn(gf, dz, acc.z);
        } else {
            acc.w = __fmaf_rn(pj.w, kernel_w_kind(C.kw, r), acc.w);
        }
    });
}

// Field pass: one thread per lattice point, x fastest.
__global__ void k_surf_field(SurfLattice L, SurfGrid g, const uint32_t* __restrict__ cstart, const float4* __restrict__ sp, float* __restrict__ phi) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t np = L.n[0] * L.n[1] * L.n[2];
    if (p >= np) return;
    const uint32_t i = p % L.n[0], j = (p / L.n[0]) % L.n[1], k = p / (L.n[0] * L.n[1]);
    float4 acc;
    surf_gather<false>(surf_coord(L, 0, i), surf_coord(L, 1, j), surf_coord(L, 2, k), g, cstart, sp, acc);
    phi[p] = acc.w;
}

__device__ __forceinline__ bool surf_inside(float phi, float iso) { return phi >= iso; }

// Per lattice point: the crossed owned edges (bit d of emask = direction d) and their count, and the triangles of the cube
// whose lowest corner the point is.  Totals are summed in 64 bits so the host can refuse a mesh past 2^32 - 1.
__global__ void k_surf_count(SurfLattice L, const float* __restrict__ phi, uint8_t* __restrict__ emask, uint32_t* __restrict__ vcnt,
                             uint32_t* __restrict__ tcnt, unsigned long long* __restrict__ totals) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n0 = L.n[0], n1 = L.n[1], n2 = L.n[2], np = n0 * n1 * n2;
    uint32_t nv = 0, nt = 0;
    if (p < np) {
        const uint32_t i = p % n0, j = (p / n0) % n1, k = p / (n0 * n1);
        const bool ok[3] = {i + 1 < n0, j + 1 < n1, k + 1 < n2};
        uint32_t in = 0;  // inside bit of the cube corner with offset bits b, for the corners inside the lattice
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const int bx = b & 1, by = (b >> 1) & 1, bz = (b >> 2) & 1;
            if ((bx && !ok[0]) || (by && !ok[1]) || (bz && !ok[2])) continue;
            if (surf_inside(phi[p + bx + n0 * (by + n1 * bz)], L.iso)) in |= 1u << b;
        }
        const uint32_t in0 = in & 1u;
        uint32_t m = 0;
#pragma unroll
        for (int d = 0; d < 7; ++d) {
            const int b = SURF_DIR_BITS[d];
            if (((b & 1) && !ok[0]) || ((b & 2) && !ok[1]) || ((b & 4) && !ok[2])) continue;
            if (((in >> b) & 1u) != in0) m |= 1u << d;
        }
        nv = __popc(m);
        emask[p] = (uint8_t)m;
        if (ok[0] && ok[1] && ok[2])
            for (int t = 0; t < 6; ++t) {
                int c = 0;
#pragma unroll
                for (int v = 0; v < 4; ++v) c |= (int)((in >> SURF_TET[t][v]) & 1u) << v;
                nt += SURF_CASES[c][0];
            }
        vcnt[p] = nv;
        tcnt[p] = nt;
    }
    unsigned long long a = nv, b = nt;
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0 && (a | b)) {
        atomicAdd(&totals[0], a);
        atomicAdd(&totals[1], b);
    }
}

// Emission: vertices at the crossed owned edges (voff: their exclusive scan), triangles of the cube (toff likewise).
__global__ void k_surf_emit(SurfLattice L, const float* __restrict__ phi, const uint8_t* __restrict__ emask, const uint32_t* __restrict__ voff,
                            const uint32_t* __restrict__ toff, float* __restrict__ verts, uint32_t* __restrict__ tris) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n0 = L.n[0], n1 = L.n[1], n2 = L.n[2], np = n0 * n1 * n2;
    if (p >= np) return;
    const uint32_t i = p % n0, j = (p / n0) % n1, k = p / (n0 * n1);
    const uint32_t m = emask[p];
    if (m) {
        uint32_t v = voff[p];
        const float pa0[3] = {surf_coord(L, 0, i), surf_coord(L, 1, j), surf_coord(L, 2, k)};
        const float f0 = phi[p];
        for (int d = 0; d < 7; ++d) {
            if (!((m >> d) & 1u)) continue;
            const int b = SURF_DIR_BITS[d];
            const uint32_t q = p + (b & 1) + n0 * (((b >> 1) & 1) + n1 * ((b >> 2) & 1));
            const float pb0[3] = {surf_coord(L, 0, i + (b & 1)), surf_coord(L, 1, j + ((b >> 1) & 1)), surf_coord(L, 2, k + ((b >> 2) & 1))};
            const float f1 = phi[q];
            const bool a_is_p = surf_inside(f0, L.iso);  // the edge is crossed: exactly one end is inside, and it is a
            const float fa = a_is_p ? f0 : f1, fb = a_is_p ? f1 : f0;
            const float* xa = a_is_p ? pa0 : pb0;
            const float* xb = a_is_p ? pb0 : pa0;
            const float t = __fdiv_rn(__fsub_rn(L.iso, fa), __fsub_rn(fb, fa));
#pragma unroll
            for (int a = 0; a < 3; ++a) verts[3 * (size_t)v + a] = __fadd_rn(xa[a], __fmul_rn(t, __fsub_rn(xb[a], xa[a])));
            ++v;
        }
    }
    if (i + 1 >= n0 || j + 1 >= n1 || k + 1 >= n2) return;
    uint32_t in = 0;
#pragma unroll
    for (int b = 0; b < 8; ++b)
        if (surf_inside(phi[p + (b & 1) + n0 * (((b >> 1) & 1) + n1 * ((b >> 2) & 1))], L.iso)) in |= 1u << b;
    if (in == 0 || in == 0xFFu) return;
    uint32_t t_out = toff[p];
    for (int t = 0; t < 6; ++t) {
        int c = 0;
        for (int v = 0; v < 4; ++v) c |= (int)((in >> SURF_TET[t][v]) & 1u) << v;
        const int nt = SURF_CASES[c][0];
        for (int r = 0; r < nt; ++r) {
            uint32_t idx[3];
            for (int e = 0; e < 3; ++e) {
                const int te = SURF_CASES[c][1 + 3 * r + e];
                const int cu = SURF_TET[t][SURF_TET_EDGE[te][0]], cv = SURF_TET[t][SURF_TET_EDGE[te][1]];
                const uint32_t owner = p + (cu & 1) + n0 * (((cu >> 1) & 1) + n1 * ((cu >> 2) & 1));
                const int d = surf_dir_index(cv ^ cu);  // cu's bits are a subset of cv's
                idx[e] = voff[owner] + __popc((uint32_t)emask[owner] & ((1u << d) - 1u));
            }
            if (SURF_TET_ODD[t]) {
                const uint32_t s = idx[1];
                idx[1] = idx[2];
                idx[2] = s;
            }
            tris[3 * (size_t)t_out] = idx[0];
            tris[3 * (size_t)t_out + 1] = idx[1];
            tris[3 * (size_t)t_out + 2] = idx[2];
            ++t_out;
        }
    }
}

// Normals: n = -grad phi / |grad phi| at every vertex, 0 where the gradient is 0.
__global__ void k_surf_normals(uint32_t nv, const float* __restrict__ verts, SurfGrid g, const uint32_t* __restrict__ cstart,
                               const float4* __restrict__ sp, float* __restrict__ nrm) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    float4 acc;
    surf_gather<true>(verts[3 * (size_t)v], verts[3 * (size_t)v + 1], verts[3 * (size_t)v + 2], g, cstart, sp, acc);
    const float n2 = dist2_exact(acc.x, acc.y, acc.z);
    const float s = n2 > 0.f ? -__frsqrt_rn(n2) : 0.f;
    nrm[3 * (size_t)v] = acc.x * s;
    nrm[3 * (size_t)v + 1] = acc.y * s;
    nrm[3 * (size_t)v + 2] = acc.z * s;
}

// ---- anisotropic kernels (Yu & Turk 2013; include/sph.h sph_world_extract_surface_anisotropic, DESIGN.md section 17) -------
struct SurfAniso {
    float lambda, kr, kn;
    uint32_t n_eps;
};

// Cyclic Jacobi rotation of the symmetric 3x3 a in the (p, q) plane; the columns of v collect the rotations.
__device__ __forceinline__ void surf_jacobi_rot(float (&a)[3][3], float (&v)[3][3], int p, int q) {
    const float apq = a[p][q];
    if (apq == 0.f) return;
    const float theta = __fdiv_rn(__fsub_rn(a[q][q], a[p][p]), __fmul_rn(2.f, apq));
    const float at = fabsf(theta);
    // t = sign(theta) / (|theta| + sqrt(theta^2 + 1)), the smaller root; 1 / (2 theta) once theta^2 would overflow
    const float t = copysignf(at > 1e18f ? __fdiv_rn(0.5f, at) : __fdiv_rn(1.f, __fadd_rn(at, __fsqrt_rn(__fmaf_rn(at, at, 1.f)))), theta);
    const float c = __frsqrt_rn(__fmaf_rn(t, t, 1.f)), s = __fmul_rn(t, c);
    const int r = 3 - p - q;  // the third index
    const float arp = a[r][p], arq = a[r][q];
    a[p][p] = __fmaf_rn(-t, apq, a[p][p]);
    a[q][q] = __fmaf_rn(t, apq, a[q][q]);
    a[p][q] = a[q][p] = 0.f;
    a[r][p] = a[p][r] = __fsub_rn(__fmul_rn(c, arp), __fmul_rn(s, arq));
    a[r][q] = a[q][r] = __fadd_rn(__fmul_rn(s, arp), __fmul_rn(c, arq));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float vp = v[k][p], vq = v[k][q];
        v[k][p] = __fsub_rn(__fmul_rn(c, vp), __fmul_rn(s, vq));
        v[k][q] = __fadd_rn(__fmul_rn(s, vp), __fmul_rn(c, vq));
    }
}

// The ellipsoids of the collected particles.  Thread s < n handles the binned particle s: the weighted sums over the
// particles of its 27 cells within h (itself included, with weight 1), taken relative to x_s; the centre x_bar; the
// covariance's eigen-decomposition by cyclic Jacobi (at most 8 sweeps); the radii.  In collected order (row perm[s]) it
// writes (x_bar, V h^3 / (a1 a2 a3)) to c4, h G as (xx, yy, zz, xy) to g4a and (xz, yz, 0, 0) to g4b, and the public rows:
// centre xyz and (e1, a1, e2, a2, e3, a3).  Thread k < np also writes the rows of collected particle k when its position is
// not finite (it was not binned): its position as centre, zero axes and a non-finite c4 that the re-binning leaves out.
__global__ void k_surf_ellipsoids(uint32_t n, uint32_t np, SurfGrid g, const uint32_t* __restrict__ cstart, const float4* __restrict__ sp,
                                  const uint32_t* __restrict__ perm, const float4* __restrict__ p4, SurfAniso P, float4* __restrict__ c4,
                                  float4* __restrict__ g4a, float4* __restrict__ g4b, float* __restrict__ o_centre, float* __restrict__ o_axes) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < np) {
        const float4 p = p4[s];
        if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) {
            c4[s] = make_float4(p.x, p.y, p.z, 0.f);
            o_centre[3 * (size_t)s] = p.x;
            o_centre[3 * (size_t)s + 1] = p.y;
            o_centre[3 * (size_t)s + 2] = p.z;
#pragma unroll
            for (int k = 0; k < 12; ++k) o_axes[12 * (size_t)s + k] = 0.f;
        }
    }
    if (s >= n) return;
    const float4 pi = sp[s];
    float sw = 0.f, m[3] = {0.f, 0.f, 0.f}, q2[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // q2: xx yy zz xy xz yz
    uint32_t cnt = 0;
    surf_for_cells(pi.x, pi.y, pi.z, g, cstart, [&](uint32_t j) {
        const float4 pj = sp[j];
        const float dx = __fsub_rn(pi.x, pj.x), dy = __fsub_rn(pi.y, pj.y), dz = __fsub_rn(pi.z, pj.z);
        const float d2 = dist2_exact(dx, dy, dz);  // the step's unfused pair test
        if (!(d2 <= C.h2)) return;
        const float q = __fdiv_rn(__fsqrt_rn(d2), C.h);
        const float wt = __fsub_rn(1.f, __fmul_rn(__fmul_rn(q, q), q));  // 1 - (r / h)^3
        const float ox = -dx, oy = -dy, oz = -dz;                          // x_j - x_i, exactly
        ++cnt;
        sw = __fadd_rn(sw, wt);
        const float wx = __fmul_rn(wt, ox), wy = __fmul_rn(wt, oy), wz = __fmul_rn(wt, oz);
        m[0] = __fadd_rn(m[0], wx);
        m[1] = __fadd_rn(m[1], wy);
        m[2] = __fadd_rn(m[2], wz);
        q2[0] = __fmaf_rn(wx, ox, q2[0]);
        q2[1] = __fmaf_rn(wy, oy, q2[1]);
        q2[2] = __fmaf_rn(wz, oz, q2[2]);
        q2[3] = __fmaf_rn(wx, oy, q2[3]);
        q2[4] = __fmaf_rn(wx, oz, q2[4]);
        q2[5] = __fmaf_rn(wy, oz, q2[5]);
    });
    const uint32_t nn = cnt - 1;  // the particle itself is among the binned ones, at distance 0
#pragma unroll
    for (int a = 0; a < 3; ++a) m[a] = __fdiv_rn(m[a], sw);  // x^w - x_i
    const float c[3] = {__fmaf_rn(P.lambda, m[0], pi.x), __fmaf_rn(P.lambda, m[1], pi.y), __fmaf_rn(P.lambda, m[2], pi.z)};
    // C = sum w d d^T / sum w - m m^T, d = x_j - x_i
    float A[3][3], V[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};
    A[0][0] = __fmaf_rn(-m[0], m[0], __fdiv_rn(q2[0], sw));
    A[1][1] = __fmaf_rn(-m[1], m[1], __fdiv_rn(q2[1], sw));
    A[2][2] = __fmaf_rn(-m[2], m[2], __fdiv_rn(q2[2], sw));
    A[0][1] = A[1][0] = __fmaf_rn(-m[0], m[1], __fdiv_rn(q2[3], sw));
    A[0][2] = A[2][0] = __fmaf_rn(-m[0], m[2], __fdiv_rn(q2[4], sw));
    A[1][2] = A[2][1] = __fmaf_rn(-m[1], m[2], __fdiv_rn(q2[5], sw));
    for (int sweep = 0; sweep < 8; ++sweep) {
        const float off = fabsf(A[0][1]) + fabsf(A[0][2]) + fabsf(A[1][2]);
        const float diag = fabsf(A[0][0]) + fabsf(A[1][1]) + fabsf(A[2][2]);
        if (!(off > 1e-7f * diag)) break;  // converged (or the matrix is 0)
        surf_jacobi_rot(A, V, 0, 1);
        surf_jacobi_rot(A, V, 0, 2);
        surf_jacobi_rot(A, V, 1, 2);
    }
    float sg[3] = {fmaxf(A[0][0], 0.f), fmaxf(A[1][1], 0.f), fmaxf(A[2][2], 0.f)};
    // descending, columns of V with them (three compare-exchanges)
    auto cx = [&](int i, int j) {
        if (sg[j] > sg[i]) {
            const float t = sg[i];
            sg[i] = sg[j];
            sg[j] = t;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float u = V[k][i];
                V[k][i] = V[k][j];
                V[k][j] = u;
            }
        }
    };
    cx(0, 1);
    cx(1, 2);
    cx(0, 1);
    float ax[3];
    if (nn >= P.n_eps && sg[0] > 0.f) {
        // h max(s_k / s1, 1 / k_r): the ratio first, so a denormal s1 / k_r cannot flatten an axis to 0
        const float lo = __fdiv_rn(1.f, P.kr);
#pragma unroll
        for (int k = 0; k < 3; ++k) ax[k] = k == 0 ? C.h : __fmul_rn(C.h, fmaxf(__fdiv_rn(sg[k], sg[0]), lo));
    } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            ax[k] = __fmul_rn(P.kn, C.h);
#pragma unroll
            for (int r = 0; r < 3; ++r) V[r][k] = r == k ? 1.f : 0.f;
        }
    }
    // h G = sum_k e_k e_k^T (h / a_k); the kernel's scale V h^3 / (a1 a2 a3)
    const float ih[3] = {__fdiv_rn(C.h, ax[0]), __fdiv_rn(C.h, ax[1]), __fdiv_rn(C.h, ax[2])};
    float G[6];
    const int gi[6] = {0, 1, 2, 0, 0, 1}, gj[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; ++e) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) acc = __fmaf_rn(__fmul_rn(V[gi[e]][k], V[gj[e]][k]), ih[k], acc);
        G[e] = acc;
    }
    const float scale = __fmul_rn(__fmul_rn(__fmul_rn(pi.w, ih[0]), ih[1]), ih[2]);
    const uint32_t o = perm[s];
    c4[o] = make_float4(c[0], c[1], c[2], scale);
    g4a[o] = make_float4(G[0], G[1], G[2], G[3]);
    g4b[o] = make_float4(G[4], G[5], 0.f, 0.f);
#pragma unroll
    for (int a = 0; a < 3; ++a) o_centre[3 * (size_t)o + a] = c[a];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int r = 0; r < 3; ++r) o_axes[12 * (size_t)o + 4 * k + r] = V[r][k];
        o_axes[12 * (size_t)o + 4 * k + 3] = ax[k];
    }
}

// u = (h G) (x - x_bar) of the binned ellipsoid j at x; |u|^2 unfused
__device__ __forceinline__ float surf_aniso_u(float x, float y, float z, float4 c, float4 ga, float4 gb, float (&u)[3]) {
    const float dx = __fsub_rn(x, c.x), dy = __fsub_rn(y, c.y), dz = __fsub_rn(z, c.z);
    u[0] = __fmaf_rn(gb.x, dz, __fmaf_rn(ga.w, dy, __fmul_rn(ga.x, dx)));
    u[1] = __fmaf_rn(gb.y, dz, __fmaf_rn(ga.y, dy, __fmul_rn(ga.w, dx)));
    u[2] = __fmaf_rn(ga.z, dz, __fmaf_rn(gb.y, dy, __fmul_rn(gb.x, dx)));
    return dist2_exact(u[0], u[1], u[2]);
}

// Anisotropic field pass: one thread per lattice point, x fastest; phi = sum_j s_j W(|u_j|) over the binned centres of the 27
// cells around the point, s_j = V_j h^3 / (a1 a2 a3).
__global__ void k_surf_field_aniso(SurfLattice L, SurfGrid g, const uint32_t* __restrict__ cstart, const float4* __restrict__ sc,
                                   const float4* __restrict__ sga, const float4* __restrict__ sgb, float* __restrict__ phi) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t np = L.n[0] * L.n[1] * L.n[2];
    if (p >= np) return;
    const uint32_t i = p % L.n[0], j = (p / L.n[0]) % L.n[1], k = p / (L.n[0] * L.n[1]);
    const float x = surf_coord(L, 0, i), y = surf_coord(L, 1, j), z = surf_coord(L, 2, k);
    float acc = 0.f;
    surf_for_cells(x, y, z, g, cstart, [&](uint32_t e) {
        const float4 c = sc[e];
        float u[3];
        const float u2 = surf_aniso_u(x, y, z, c, sga[e], sgb[e], u);
        if (!(u2 <= C.h2)) return;
        acc = __fmaf_rn(c.w, kernel_w_kind(C.kw, __fsqrt_rn(u2)), acc);
    });
    phi[p] = acc;
}

// Anisotropic normals: n = -grad phi / |grad phi|, grad W_j = s_j (h G_j) W'(|u|) / |u| u (0 for |u|^2 <= eps^2), 0 where the
// gradient is 0 (k_surf_normals' rule).
__global__ void k_surf_normals_aniso(uint32_t nv, const float* __restrict__ verts, SurfGrid g, const uint32_t* __restrict__ cstart,
                                     const float4* __restrict__ sc, const float4* __restrict__ sga, const float4* __restrict__ sgb,
                                     float* __restrict__ nrm) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    const float x = verts[3 * (size_t)v], y = verts[3 * (size_t)v + 1], z = verts[3 * (size_t)v + 2];
    float acc[3] = {0.f, 0.f, 0.f};
    surf_for_cells(x, y, z, g, cstart, [&](uint32_t e) {
        const float4 c = sc[e], ga = sga[e], gb = sgb[e];
        float u[3];
        const float u2 = surf_aniso_u(x, y, z, c, ga, gb, u);
        if (!(u2 <= C.h2) || !(u2 > F32_EPS * F32_EPS)) return;
        const float r = __fsqrt_rn(u2);
        const float gf = __fmul_rn(c.w, __fdiv_rn(kernel_dw_kind(C.kg, r), r));
        const float t[3] = {__fmul_rn(gf, u[0]), __fmul_rn(gf, u[1]), __fmul_rn(gf, u[2])};
        acc[0] = __fadd_rn(acc[0], __fmaf_rn(gb.x, t[2], __fmaf_rn(ga.w, t[1], __fmul_rn(ga.x, t[0]))));
        acc[1] = __fadd_rn(acc[1], __fmaf_rn(gb.y, t[2], __fmaf_rn(ga.y, t[1], __fmul_rn(ga.w, t[0]))));
        acc[2] = __fadd_rn(acc[2], __fmaf_rn(ga.z, t[2], __fmaf_rn(gb.y, t[1], __fmul_rn(gb.x, t[0]))));
    });
    const float n2 = dist2_exact(acc[0], acc[1], acc[2]);
    const float s = n2 > 0.f ? -__frsqrt_rn(n2) : 0.f;
    nrm[3 * (size_t)v] = acc[0] * s;
    nrm[3 * (size_t)v + 1] = acc[1] * s;
    nrm[3 * (size_t)v + 2] = acc[2] * s;
}

}  // namespace sphk
