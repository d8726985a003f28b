// sph_kernels.cuh — sm_90a CUDA kernels of the SPH step path.
//
// Data layout (all per-particle arrays are in SORTED order: x-major cell order, z fastest, so the
// 27-cell stencil of a particle is 9 contiguous runs of the sorted arrays):
//   pos4  : x, y, z, mass          (mass = volume * density0 of the particle's fluid, fluid.rs:183-185)
//   vel4  : vx, vy, vz, fluid id   (bit pattern of the fluid index in .w)
//   vc4   : velocity_changes       (dfsph_solver.rs:44)
//   vs4   : v* = vel + vc          (materialised so gather passes read ONE vector per neighbour)
//   bpos4 : boundary x, y, z, volume (dfsph_solver.rs:72-96);  bvel4: boundary velocity, boundary id
// The neighbour lists' layout is sph_lists.cuh's.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <climits>

namespace sphk {

constexpr int MAX_FLUIDS = 16;
constexpr int MAX_BOUNDARIES = 64;
constexpr float F32_EPS = 1.1920929e-07f;

struct FluidParams {  // per fluid, in __constant__ memory
    float density0;
    uint32_t memberships, filter;
    float mass;  // the particles' common mass when every particle of the fluid has the same volume, else 0
};
struct BoundaryParams {
    uint32_t memberships, filter;
};
struct Consts {
    float h, inv_h, h2;          // h2 = h*h rounded once (contacts.rs:285 `h * h`)
    float sigma;                 // 8 / (pi h^3)            cubic_spline_kernel.rs:18
    float dsigma;                // sigma / h               cubic_spline_kernel.rs:79
    float dsigma6;               // 6 sigma / h
    float g_t2;                  // gradient is zero unless |x_ij|^2 > g_t2 = max(eps^2, (1e-5 h)^2)  (kernel.rs:19 + cubic_spline_kernel.rs:64)
    // DFSPHSolver<KernelDensity, KernelGradient> / IISPHSolver<..> type parameters (dfsph_solver.rs:17-20): 0 = CubicSpline
    // (default, the lean path), 1 = Poly6, 2 = Spiky, 3 = Viscosity; kgen != 0 <=> any of the two is not the cubic spline
    int kw, kg, kgen;
    float poly6_n, spiky_n, visc_n;  // 315/(64 pi h^9), 15/(pi h^6), 15/(2 pi h^3)
    int ox, oy, oz;              // grid origin in cell coordinates (one padding cell each side)
    int nx, ny, nz;
    float h_reach;               // h * (1 + 1e-5): covers every |dx| the f32 test d^2 <= h^2 can accept (row order, arun())
    // "row order" (SALVA_B200_XYSUB, one GPU): x and y are binned `xysub` times finer than h (ox, oy, nx, ny then
    // count BINS), z stays the run direction.  With xysub = 2 and the usual spacing h/2 every (x, y) bin column holds ONE line of
    // particles along z, so the 32 lanes of a warp are 32 consecutive particles of a line and their k-th contacts are consecutive
    // particles of a neighbouring line: a warp-wide gather touches ~4 cache lines instead of ~17 data-pipe wavefronts
    // (tools/sim_gather_order.py models this).  Contact SETS are unchanged (k_neighbors_xy clips its rows, see arun()).
    int xysub;
    float xysub_f;
    uint32_t n_fluid, n_bound;   // particle totals (n_fluid counts owned + ghost slots of the sorted arrays)
    uint32_t i_begin, n_owned;   // owned slots [i_begin, i_begin + n_owned): everything on one GPU; the slab between the
                                 // two ghost columns in a multi-GPU world (x-major order keeps ghosts at both ends)
    uint32_t stride;             // the world's per-particle plane stride (>= n_fluid, multiple of 32): neighbour-list rows,
                                 // DFSPHViscosity's beta / target planes
    uint32_t cap_f, cap_b;       // neighbour-list capacities (rows)
    int n_fluids, n_bounds;      // object counts
    FluidParams fluids[MAX_FLUIDS];
    BoundaryParams bounds[MAX_BOUNDARIES];
};

__constant__ Consts C;

}  // namespace sphk

#include "sph_lists.cuh"
#include "sph_order.cuh"

namespace sphk {

// ------------------------------------------------------------------------------------------------
// geometry helpers
// ------------------------------------------------------------------------------------------------
// hgrid.rs:41-52: cell = floor(x / h), IEEE division exactly as the reference.
__device__ __forceinline__ int cell_coord(float x) { return (int)floorf(__fdiv_rn(x, C.h)); }

// A cell-coordinate AABB (lo, hi inclusive; lo > hi on an axis without a point) and whether a point had a coordinate without
// a cell.  The dense grid covers the fluid's and the boundaries' boxes.
struct CellBox {
    int lo[3], hi[3];
    int bad;
};
constexpr CellBox CELL_BOX_EMPTY{{INT_MAX, INT_MAX, INT_MAX}, {INT_MIN, INT_MIN, INT_MIN}, 0};

// Adds the point (x, y, z) to b: its cell is floor(x / h) with IEEE division (cell_coord) on the device and on the host alike;
// a coordinate whose cell is NaN, infinite or absurd (|cell| >= 1e9) sets bad instead.
__host__ __device__ __forceinline__ void cell_box_add(CellBox& b, float x, float y, float z, float h) {
#ifdef __CUDA_ARCH__
    const float c[3] = {floorf(__fdiv_rn(x, h)), floorf(__fdiv_rn(y, h)), floorf(__fdiv_rn(z, h))};
#else
    const float c[3] = {floorf(x / h), floorf(y / h), floorf(z / h)};
#endif
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (!(fabsf(c[a]) < 1.0e9f)) { b.bad = 1; continue; }
        b.lo[a] = (int)c[a] < b.lo[a] ? (int)c[a] : b.lo[a];
        b.hi[a] = (int)c[a] > b.hi[a] ? (int)c[a] : b.hi[a];
    }
}
inline void merge(CellBox& b, const CellBox& o) {
    for (int a = 0; a < 3; ++a) {
        b.lo[a] = std::min(b.lo[a], o.lo[a]);
        b.hi[a] = std::max(b.hi[a], o.hi[a]);
    }
    b.bad |= o.bad;
}

// The warp's boxes merged into every lane's b
__device__ __forceinline__ void cell_box_warp_reduce(CellBox& b) {
#pragma unroll
    for (int a = 0; a < 3; ++a)
        for (int o = 16; o > 0; o >>= 1) {
            b.lo[a] = min(b.lo[a], __shfl_xor_sync(0xffffffffu, b.lo[a], o));
            b.hi[a] = max(b.hi[a], __shfl_xor_sync(0xffffffffu, b.hi[a], o));
        }
    b.bad = __any_sync(0xffffffffu, b.bad);
}
// Merges the warp's boxes into *out with one global atomic per axis and bound from lane 0.  Every lane of the warp calls it.
__device__ __forceinline__ void cell_box_commit_warp(CellBox b, CellBox* out) {
    cell_box_warp_reduce(b);
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (b.lo[a] <= b.hi[a]) {
                atomicMin(&out->lo[a], b.lo[a]);
                atomicMax(&out->hi[a], b.hi[a]);
            }
        if (b.bad) atomicOr(&out->bad, 1);
    }
}
// Merges the block's boxes into *out: warp shuffles, then shared memory, then one global atomic per axis and bound per block
// (a kernel with one thread per particle would otherwise issue eight times as many).  Every thread of the block (at most 256)
// calls it; it contains a block barrier.
__device__ __forceinline__ void cell_box_commit_block(CellBox b, CellBox* out) {
    cell_box_warp_reduce(b);
    __shared__ int s_lo[3][8], s_hi[3][8], s_bad[8];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            s_lo[a][wid] = b.lo[a];
            s_hi[a][wid] = b.hi[a];
        }
        s_bad[wid] = b.bad;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        const int a = threadIdx.x, nw = (blockDim.x + 31) >> 5;
        int m0 = INT_MAX, m1 = INT_MIN;
#pragma unroll 4  // unrolled 8 times, the loads of all warps' entries lift k_edit_classify from 28 to 31 registers
        for (int k = 0; k < nw; ++k) {
            m0 = min(m0, s_lo[a][k]);
            m1 = max(m1, s_hi[a][k]);
        }
        if (m0 <= m1) {
            atomicMin(&out->lo[a], m0);
            atomicMax(&out->hi[a], m1);
        }
        if (a == 0) {
            int bad = 0;
            for (int k = 0; k < nw; ++k) bad |= s_bad[k];
            if (bad) atomicOr(&out->bad, 1);
        }
    }
}

// The bits of StepScalars::err.  The host tells them apart: a zero density or boundary-volume denominator (the boundary
// volumes are checked right after the search, the passes at the end of the step), a ghost exchange that timed out, and a zero
// density found by the search's density sweep (reported with the passes' zero densities).
enum : int { ERR_ZERO_DENSITY = 1, ERR_PEER_TIMEOUT = 2, ERR_SEARCH_ZERO_DENSITY = 4 };

// What the step reads back from the device: one block (sph_world::d_ss) and its pinned host mirror (sph_world::h_ss).  The
// fields are ordered so that each reset is one range: a substep of the host path sets grid .. contacts_f (phase_grid), a
// graph step zeroes err .. contacts_f; the host path reads err .. next back with one copy at the end of a substep.
struct StepScalars {
    CellBox grid;                    // the fluid's cell box that sizes the grid (k_bounds)
    int err;                         // error word: ERR_* bits
    uint32_t max_nb[3];              // the widest fluid [0] and boundary [1] contact list of the search; [2] != 0: a narrow
                                     // search met a stencil window of more than WINDOW_SLOTS slots (sph_lists.cuh)
    unsigned long long contacts_bb;  // boundary-boundary contacts (k_boundary_volumes)
    unsigned long long contacts_f;   // fluid-fluid + fluid-boundary contacts (k_sum_u32)
    uint32_t elast_width;            // the widest Becker2009 rest list (k_el_capture_lists)
    uint32_t cfl_bits;               // the CFL maximum |v + a R|^2 as float bits (k_cfl_max)
    CellBox next;                    // the cell box of the positions the step wrote (k_update_positions)
    float loop_err[MAX_FLUIDS];      // per-fluid error sums of a Jacobi evaluation (k_reduce_partials)
};

__device__ __forceinline__ int cell_id(int cx, int cy, int cz) { return ((cx - C.ox) * C.ny + (cy - C.oy)) * C.nz + (cz - C.oz); }
// Row order bins x / y `sub` times finer than h.  abin: reference cell floor(v / h) (same IEEE division) times sub plus the
// slice inside the cell.  Monotone non-decreasing in v (correctly rounded division, exact q - floor(q)), and every bin lies
// inside ONE reference cell.
__device__ __forceinline__ int abin(float v, int sub, float subf) {
    const float q = __fdiv_rn(v, C.h), fl = floorf(q);
    return (int)fl * sub + min(sub - 1, (int)((q - fl) * subf));
}
// Bins [lo, hi] a particle at v (reference cell c) has to scan: everything within h_reach of v, clipped to the three reference
// cells c-1..c+1 the reference's 27-cell stencil looks at.  A pair that passes the f32 test (dx^2 + dy^2) + dz^2 <= h^2 has
// |v_i - v_j| <= h (1 + 2^-22) < h_reach; the bounds are rounded outwards, and abin is monotone, so no accepted pair of
// adjacent reference cells is ever cut off: the contact sets stay exactly the reference's.
__device__ __forceinline__ void arun(float v, int c, int sub, float subf, int& lo, int& hi) {
    lo = max(abin(__fsub_rd(v, C.h_reach), sub, subf), (c - 1) * sub);
    hi = min(abin(__fadd_ru(v, C.h_reach), sub, subf), (c + 2) * sub - 1);
}

// contacts.rs:285,322,366: (dx*dx + dy*dy) + dz*dz <= h*h with no contraction (rustc never fuses).
__device__ __forceinline__ float dist2_exact(float dx, float dy, float dz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// cubic_spline_kernel.rs:12-33: W(r) for q = r/h.
__device__ __forceinline__ float kernel_w(float r) {
    float q = r * C.inv_h;
    float q2 = q * q;
    float a = 1.0f + (q2 * q - q2) * 6.0f;
    float t = 1.0f - q;
    float b = (t * t * t) * 2.0f;
    float rhs = q <= 0.5f ? a : (q <= 1.0f ? b : 0.0f);
    return C.sigma * rhs;
}
// MUFU.RSQ without the denormal-rescue sequence rsqrtf() compiles to (3 extra instructions per contact): operands
// here are squared distances floored at 1e-30, far above the denormals.
__device__ __forceinline__ float rsqrt_ftz(float x) {
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// kernel/poly6_kernel.rs:12-40, spiky_kernel.rs:12-40, viscosity_kernel.rs:12-51 (dim3), evaluated like the reference
// (IEEE sqrt / division, powi as repeated products); kind 0 falls through to the cubic spline.
__device__ __forceinline__ float kernel_w_kind(int kind, float r) {
    const float h = C.h;
    if (kind == 1) {
        const float t = h * h - r * r;
        return r <= h ? C.poly6_n * (t * t * t) : 0.f;
    }
    if (kind == 2) {
        const float t = h - r;
        return r <= h ? C.spiky_n * (t * t * t) : 0.f;
    }
    if (kind == 3) {
        if (!(r > 0.f && r <= h)) return 0.f;
        const float rr_hh = __fdiv_rn(r * r, h * h);
        return C.visc_n * (rr_hh * (1.0f - __fdiv_rn(r, 2.0f * h)) + __fdiv_rn(h, 2.0f * r) - 1.0f);
    }
    return kernel_w(r);
}
__device__ __forceinline__ float kernel_dw_kind(int kind, float r) {  // scalar_apply_diff
    const float h = C.h;
    if (kind == 1) {
        const float t = h * h - r * r;
        return r <= h ? C.poly6_n * (t * t) * r * -6.0f : 0.f;
    }
    if (kind == 2) {
        const float t = h - r;
        return r <= h ? -C.spiky_n * (t * t) * 3.0f : 0.f;
    }
    if (kind == 3) {
        if (!(r > 0.f && r <= h)) return 0.f;
        const float rr = r * r, hh = h * h;
        return C.visc_n * (__fdiv_rn(-3.0f * rr, 2.0f * (hh * h)) + __fdiv_rn(2.0f * r, hh) - __fdiv_rn(h, 2.0f * rr));
    }
    const float q = __fdiv_rn(r, h);  // cubic_spline_kernel.rs:55-80
    const float t = 1.0f - q;
    const float rhs = (q > 1.0f || q <= 1.0e-5f) ? 0.f : (q <= 0.5f ? (q * 3.0f - 2.0f) * q * 6.0f : -t * t * 6.0f);
    return __fdiv_rn(C.sigma * rhs, h);
}

// The solver's KernelDensity / KernelGradient are COMPILE-TIME type parameters in the reference (monomorphised per solver
// type).  Here likewise: libsalva_b200.so is built with SPH_GENERIC_KERNELS = 0 (cubic spline only, no branch in the pair
// evaluation: a uniform `if (C.kgen)` inside the 4-way unrolled contact loops costs every step); libsalva_b200_kernels.so is the same source built with SPH_GENERIC_KERNELS = 1 and
// serves worlds whose solver names Poly6 / Spiky / Viscosity kernels.  Same C ABI in both.
#ifndef SPH_GENERIC_KERNELS
#define SPH_GENERIC_KERNELS 0
#endif
__device__ __forceinline__ float2 pair_generic(float d2, int need_w, int need_g) {
    const float r = __fsqrt_rn(d2);
    float2 o;
    o.x = need_w ? kernel_w_kind(C.kw, r) : 0.f;
    o.y = (need_g && d2 > F32_EPS * F32_EPS) ? __fdiv_rn(kernel_dw_kind(C.kg, r), r) : 0.f;
    return o;
}

struct Pair {        // geometry of one (i, j) contact
    float dx, dy, dz;  // x_i - x_j
    float d2, r;
    float w;           // contact.weight
    float g;           // contact.gradient = g * (dx, dy, dz)
};
// CUBIC_ONLY: force plugins with their OWN kernel type parameters (Becker2009Elasticity<CubicSplineKernel, ..>) do not
// follow the solver's kernels.
template <bool NEED_W, bool NEED_G, bool CUBIC_ONLY = false>
__device__ __forceinline__ Pair make_pair(const float4& pi, const float4& pj) {
    Pair p;
    p.dx = pi.x - pj.x;
    p.dy = pi.y - pj.y;
    p.dz = pi.z - pj.z;
    p.d2 = fmaf(p.dz, p.dz, fmaf(p.dy, p.dy, p.dx * p.dx));
    if (SPH_GENERIC_KERNELS && !CUBIC_ONLY && C.kgen) {  // non-default solver kernels: uniform branch, off the default path
        const float2 o = pair_generic(p.d2, NEED_W, NEED_G);
        p.r = __fsqrt_rn(p.d2);
        p.w = o.x;
        p.g = o.y;
        return p;
    }
    // Contacts come from lists built with d^2 <= h^2, so q <= 1 up to rounding (where (1 - q)^2 ~ 1e-14 anyway), and the
    // two "zero gradient" guards of the reference (|x_ij|^2 > eps^2, q > 1e-5) collapse into one select on d2.  r itself
    // is the distance down to d2 = 0 (the floor keeps rsqrt finite, so 0 * inv_r = 0): Akinci2013's cohesion and adhesion
    // act on every pair with |x_ij|^2 > eps^2, below the gradient's threshold too, and divide by r.  W takes the true r as
    // well; at q <= 1e-5, 1 - 6 q^2 rounds to 1 as it did with r = 0.
    const float inv_r = rsqrt_ftz(fmaxf(p.d2, 1.0e-30f));
    const bool nz = p.d2 > C.g_t2;
    p.r = p.d2 * inv_r;
    const float q = p.r * C.inv_h;
    const float t = 1.0f - q;
    const bool inner = q <= 0.5f;
    if (NEED_W) {
        const float q2 = q * q;
        const float a = fmaf(fmaf(q2, q, -q2), 6.0f, 1.0f);
        const float b = (t * t) * (t * 2.0f);
        p.w = C.sigma * (inner ? a : b);
    } else {
        p.w = 0.f;
    }
    if (NEED_G) {
        const float a = fmaf(q, 3.0f, -2.0f) * q;
        const float b = -t * t;
        p.g = nz ? (C.dsigma6 * inv_r) * (inner ? a : b) : 0.f;
    } else {
        p.g = 0.f;
    }
    return p;
}

// index of the owned particle handled by this thread (returns from the kernel when out of range)
#define SPH_OWNED_INDEX(i)                                   \
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;      \
    if (i >= C.n_owned) return;                              \
    i += C.i_begin;

__device__ __forceinline__ uint32_t fid_of(const float4& v) { return __float_as_uint(v.w); }

// interaction_groups.rs:64-69
__device__ __forceinline__ bool groups_test(uint32_t m1, uint32_t f1, uint32_t m2, uint32_t f2) {
    return (m1 & f2) != 0 && (m2 & f1) != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Deterministic block sum (fixed tree); result valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* sm /* >= 32 floats */) {
    v = warp_sum(v);
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sm[wid] = v;
    __syncthreads();
    if (wid == 0) {
        int nw = (blockDim.x + 31) >> 5;
        v = lane < nw ? sm[lane] : 0.f;
        v = warp_sum(v);
    }
    return v;
}

// ------------------------------------------------------------------------------------------------
// K0: bounds (cell-coordinate AABB) — replaces the unbounded HashMap of hgrid.rs:22-25 by a dense
// grid over the occupied region.
// ------------------------------------------------------------------------------------------------
__global__ void k_bounds(const float4* __restrict__ pos, uint32_t n, CellBox* __restrict__ out) {
    CellBox b = CELL_BOX_EMPTY;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = pos[i];
        cell_box_add(b, p.x, p.y, p.z, C.h);
    }
    cell_box_commit_block(b, out);
}

// ------------------------------------------------------------------------------------------------
// K1: counting sort by cell (replaces HGrid::insert hgrid.rs:60-63 / insert_*_to_grid contacts.rs:133-151
// and the dead z_order.rs sort).
// ------------------------------------------------------------------------------------------------
// In-cell ranks take one atomic per distinct cell of a warp (__match_any_sync), and follow input order within the warp.  The
// input is usually the previous step's sorted order, so most cells leave the scatter already in canonical order and the
// sort below only fixes what the order of the warps' atomics shuffled.  live == false (a tail lane or a dead slot) takes no rank.
__device__ __forceinline__ uint32_t warp_cell_rank(uint32_t id, bool live, uint32_t* __restrict__ count) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t peers = __match_any_sync(0xffffffffu, live ? id : 0xFFFFFFFFu);
    const uint32_t leader = __ffs(peers) - 1u;
    uint32_t base = 0u;
    if (live && lane == leader) base = atomicAdd(&count[id], (uint32_t)__popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    return base + __popc(peers & ((1u << lane) - 1u));
}

// dead (optional): dead[i] != 0 for i < n_dead marks an input slot that must not enter the sorted arrays (a particle that left
// this rank's slab, sph_slab.inl); such slots get cid = 0xFFFFFFFF and are skipped by the scatter.
// Every lane of a warp runs to the rank (no early return): __match_any_sync takes the whole warp.
__global__ void k_cell_hist(const float4* __restrict__ pos, uint32_t n, uint32_t* __restrict__ cid, uint32_t* __restrict__ rank,
                            uint32_t* __restrict__ count, const uint32_t* __restrict__ dead, uint32_t n_dead) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < n;
    const bool live = in && !(dead && i < n_dead && dead[i]);
    uint32_t id = 0xFFFFFFFFu;
    if (live) {
        const float4 p = pos[i];
        id = (uint32_t)cell_id(cell_coord(p.x), cell_coord(p.y), cell_coord(p.z));
    }
    const uint32_t r = warp_cell_rank(id, live, count);
    if (!in) return;
    cid[i] = id;
    if (live) rank[i] = r;
}

// row order (Consts::xysub > 1): x and y binned finer than h
__global__ void k_cell_hist_xy(const float4* __restrict__ pos, uint32_t n, uint32_t* __restrict__ cid, uint32_t* __restrict__ rank,
                               uint32_t* __restrict__ count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    uint32_t id = 0xFFFFFFFFu;
    if (live) {
        const float4 p = pos[i];
        id = (uint32_t)cell_id(abin(p.x, C.xysub, C.xysub_f), abin(p.y, C.xysub, C.xysub_f), cell_coord(p.z));
    }
    const uint32_t r = warp_cell_rank(id, live, count);
    if (!live) return;
    cid[i] = id;
    rank[i] = r;
}

// Deterministic mode: atomics hand out in-cell ranks in arbitrary order; k_cell_sort sorts each cell's slice of perm so the
// sorted order (and every f32 summation order downstream) is reproducible.  The in-cell order is CANONICAL — ascending
// (fluid, particle id), ties by source slot, a pure function of the particle set — so a world restored from a snapshot, a
// world whose state went through the host, and the ranks of a slab decomposition (ghost columns!) all see the same order and
// produce bit-identical sums.  Boundaries pass their original indices (borig) as the key, so their in-cell order is insertion
// order whether the input is a fresh upload or a sort of boundaries that colliders moved on the device.
__device__ __forceinline__ unsigned long long sort_key(uint32_t src, const uint32_t* __restrict__ gid, const float4* __restrict__ vel) {
    const uint32_t f = vel ? fid_of(vel[src]) : 0u;
    return ((unsigned long long)f << 32) | gid[src];
}
// key (optional, deterministic mode): each entry's sort key beside perm, so the in-cell sort reads keys contiguously instead of
// through gid[perm[.]].  gid / vel as for sort_key.
__global__ void k_cell_scatter(uint32_t n, const uint32_t* __restrict__ cid, const uint32_t* __restrict__ rank,
                               const uint32_t* __restrict__ start, uint32_t* __restrict__ perm, const uint32_t* __restrict__ gid = nullptr,
                               const float4* __restrict__ vel = nullptr, unsigned long long* __restrict__ key = nullptr) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t c = cid[i];
    if (c == 0xFFFFFFFFu) return;
    const uint32_t d = start[c] + rank[i];
    perm[d] = i;
    if (key) key[d] = sort_key(i, gid, vel);
}

// Insertion sort of each cell's slice by (key, source slot).  The largest entry so far stays in registers, so an entry already
// in place costs one load of its key and slot and one compare; keys move with their slots.
__global__ void k_cell_sort(uint32_t ncell, const uint32_t* __restrict__ start, uint32_t* __restrict__ perm, unsigned long long* __restrict__ key) {
    uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncell) return;
    const uint32_t s = start[c], e = start[c + 1];
    if (e - s < 2u) return;
    unsigned long long kt = key[s];
    uint32_t ut = perm[s];
    for (uint32_t a = s + 1; a < e; ++a) {
        const uint32_t v = perm[a];
        const unsigned long long kv = key[a];
        if (kt < kv || (kt == kv && ut < v)) {
            kt = kv;
            ut = v;
            continue;
        }
        perm[a] = ut;
        key[a] = kt;
        uint32_t b = a - 1;
        while (b > s) {
            const uint32_t u = perm[b - 1];
            const unsigned long long ku = key[b - 1];
            if (ku < kv || (ku == kv && u < v)) break;
            perm[b] = u;
            key[b] = ku;
            --b;
        }
        perm[b] = v;
        key[b] = kv;
    }
}

struct GatherSet {  // arrays reordered together by the counting sort
    const float4* in4[6];
    float4* out4[6];
    const uint32_t* in1[4];
    uint32_t* out1[4];
    int n4, n1;
};
__global__ void k_gather(uint32_t n, const uint32_t* __restrict__ perm, GatherSet g) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    uint32_t src = perm[s];
#pragma unroll
    for (int a = 0; a < 6; ++a)
        if (a < g.n4) g.out4[a][s] = g.in4[a][src];
#pragma unroll
    for (int a = 0; a < 4; ++a)
        if (a < g.n1) g.out1[a][s] = g.in1[a][src];
}

// exclusive scan, 2048 items per block (256 threads x 8)
constexpr int SCAN_T = 256, SCAN_I = 8, SCAN_B = SCAN_T * SCAN_I;
__global__ void k_scan_block(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint32_t n, uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t warp_tot[SCAN_T / 32];
    uint32_t base = blockIdx.x * SCAN_B + threadIdx.x * SCAN_I;
    uint32_t v[SCAN_I];
    uint32_t tsum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_I; ++k) {
        v[k] = (base + k < n) ? in[base + k] : 0u;
        tsum += v[k];
    }
    uint32_t incl = tsum;
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < SCAN_T / 32 ? warp_tot[lane] : 0u;
        uint32_t wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        if (lane < SCAN_T / 32) warp_tot[lane] = wi - w;
        if (lane == SCAN_T / 32 - 1 && block_sums) block_sums[blockIdx.x] = wi;
    }
    __syncthreads();
    uint32_t run = warp_tot[wid] + incl - tsum;
#pragma unroll
    for (int k = 0; k < SCAN_I; ++k) {
        if (base + k < n) out[base + k] = run;
        run += v[k];
    }
}
__global__ void k_scan_add(uint32_t* __restrict__ out, uint32_t n, const uint32_t* __restrict__ block_offsets) {
    uint32_t i = blockIdx.x * SCAN_B + threadIdx.x;
    uint32_t off = block_offsets[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_I; ++k) {
        uint32_t j = i + k * SCAN_T;
        if (j < n) out[j] += off;
    }
}

// K-way exclusive scan: the same 2048-item blocks, K independent arrays scanned by one launch (slab prologue: the five
// classification flag arrays are compacted together instead of by five 3-kernel scans).
template <int K>
struct ScanSet {
    uint32_t* a[K];
};
template <int K>
__global__ void k_scanK_block(ScanSet<K> io, uint32_t n, ScanSet<K> block_sums) {
    __shared__ uint32_t warp_tot[K][SCAN_T / 32];
    const uint32_t base = blockIdx.x * SCAN_B + threadIdx.x * SCAN_I;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < K; ++a) {
        uint32_t v[SCAN_I];
        uint32_t tsum = 0;
#pragma unroll
        for (int k = 0; k < SCAN_I; ++k) {
            v[k] = (base + k < n) ? io.a[a][base + k] : 0u;
            tsum += v[k];
        }
        uint32_t incl = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[a][wid] = incl;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = lane < SCAN_T / 32 ? warp_tot[a][lane] : 0u;
            uint32_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            if (lane < SCAN_T / 32) warp_tot[a][lane] = wi - w;
            if (lane == SCAN_T / 32 - 1 && block_sums.a[a]) block_sums.a[a][blockIdx.x] = wi;
        }
        __syncthreads();
        uint32_t run = warp_tot[a][wid] + incl - tsum;
#pragma unroll
        for (int k = 0; k < SCAN_I; ++k) {
            if (base + k < n) io.a[a][base + k] = run;
            run += v[k];
        }
    }
}
template <int K>
__global__ void k_scanK_add(ScanSet<K> io, uint32_t n, ScanSet<K> block_offsets) {
    uint32_t i = blockIdx.x * SCAN_B + threadIdx.x;
#pragma unroll
    for (int a = 0; a < K; ++a) {
        uint32_t off = block_offsets.a[a][blockIdx.x];
#pragma unroll
        for (int k = 0; k < SCAN_I; ++k) {
            uint32_t j = i + k * SCAN_T;
            if (j < n) io.a[a][j] += off;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K2: neighbour search (contacts.rs:154-400).  One thread per particle walks the 9 z-runs of its
// 27-cell stencil and keeps the indices that pass the reference's exact `d^2 <= h*h` test.
// Only ~15 % of the candidates pass, but in a warp SOME lane passes for nearly every candidate, so a store inside the
// candidate loop is executed (predicated off) by the whole warp almost every iteration.  The candidate loop therefore
// only records hits in a 32-bit mask per chunk of 32 candidates; the (short) emit loop then walks the set bits in
// ascending order, which keeps every list in the same order as a plain scan.
// BATCH4 issues the candidate loads four at a time into distinct registers (left to itself, ptxas reuses one register
// quadruple and every load waits for the previous test).  That pays on h-cell runs (~24 candidates); on the ~6-candidate runs of
// row order the plain unrolled loop is faster (C2 rows: 0.289 vs 0.304 ms per search, H100 80GB HBM3, 700 W, 1980 MHz).
// ------------------------------------------------------------------------------------------------
template <bool BATCH4, class Accept, class Emit>
__device__ __forceinline__ void scan_run(const float4& pi, const float4* __restrict__ P, uint32_t s, uint32_t e, Accept accept, Emit emit) {
    // d2 <= h*h  <=>  the sign bit of (h*h - d2) is clear (a float difference is zero only for equal operands; NaN positions
    // never get here, k_bounds rejects them): shift that bit into the mask with one funnel shift
    const auto test = [&](const float4& pj, uint32_t rej) {
        const float d2 = dist2_exact(pi.x - pj.x, pi.y - pj.y, pi.z - pj.z);
        return __funnelshift_l(__float_as_uint(__fsub_rn(C.h2, d2)), rej, 1);
    };
    for (uint32_t base = s; base < e; base += 32u) {
        const uint32_t n = min(32u, e - base);
        const float4* __restrict__ q = P + base;
        const float4* const qe = q + n;
        uint32_t rej = 0u;  // candidate t of the chunk ends up in bit n - 1 - t; set = rejected
        if (BATCH4) {
            for (; q + 4 <= qe; q += 4) {  // the four loads go out back to back, before the first test waits on one
                const float4 p0 = __ldg(q), p1 = __ldg(q + 1), p2 = __ldg(q + 2), p3 = __ldg(q + 3);
                rej = test(p3, test(p2, test(p1, test(p0, rej))));
            }
            for (; q < qe; ++q) rej = test(__ldg(q), rej);
        } else {
#pragma unroll 4
            for (; q < qe; ++q) rej = test(__ldg(q), rej);
        }
        uint32_t m = ~rej & (n == 32u ? 0xffffffffu : (1u << n) - 1u);
        while (m) {
            const uint32_t b = 31u - (uint32_t)__clz((int)m);  // highest set bit = earliest candidate
            m &= ~(1u << b);
            const uint32_t j = base + (n - 1u - b);
            if (accept(j)) emit(j);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K3 + first K4a (DFSPH), run by the neighbour search over the lists it has just built: densities (dfsph_solver.rs:628-665),
// alphas (dfsph_solver.rs:165-216) and the first compute_divergences evaluation of divergence_solve (dfsph_solver.rs:474-480).
// That evaluation reads the same neighbour positions and the step-start v* = vel + vc, and needs alpha_i only for
// kappa_i = div_i * alpha_i at the very end, so it rides along with the density.  The search holds the first NBR_SF / NBR_SB
// entries of each list in shared memory and the neighbour positions it has just streamed are still in L2, so the lists do not
// make a round trip through HBM and the step has one neighbour sweep less.  The sweep runs after the walk, whose registers are
// then dead (the kernel needs the larger of the two register sets, not their sum).  Per quantity the arithmetic and the order
// of the terms are those of a separate pass: fluid contacts in list order, then boundary contacts in list order.
// UNI: uniform-mass packed records (positions from pvx4, v* from pvx4.w + vyz2), else pos4 / vs4.
// ------------------------------------------------------------------------------------------------
constexpr int NBR_T = 128;                   // threads per block of k_neighbors / k_neighbors_xy
struct DensArgs {
    const float4* posrec;                        // pos4, or pvx4 (UNI)
    cudaTextureObject_t tposrec;                 // UNI: texture over pvx4
    const float4* vs;                            // v*
    cudaTextureObject_t tvs;                     // !UNI: texture over vs
    const float2* vyz;                           // UNI: v*.yz
    cudaTextureObject_t tvyz;                    // UNI: texture over vyz
    float *dens, *alpha, *divv, *kappa;
    float4* pk4;                                 // UNI: (position, kappa)
    float* partial;                              // per-block error partials: partial[block * n_fluids + f]
    int* err;                                    // StepScalars::err: ERR_SEARCH_ZERO_DENSITY
};
struct Vel3 {
    float x, y, z;
};
// `group(q)` returns fluid entries 4q .. 4q+3 of particle i, `bentry(k)` boundary entry k; nf / nb are the contact counts.
// Every thread of the block calls this; `valid` marks the owned ones.  `arrived` counts the block's finished warps and is 0
// on entry (the caller zeroes it before the walk).
template <bool MULTI, bool UNI, class Group, class BEntry>
__device__ __forceinline__ void density_alpha_div(uint32_t i, bool valid, uint32_t nf, uint32_t nb, const float4* __restrict__ vel,
                                                  const float4* __restrict__ bpos, const DensArgs& D, uint32_t& arrived, Group group,
                                                  BEntry bentry) {
    float e = 0.f;
    uint32_t fi = 0;
    if (valid) {
        const float4 a = D.posrec[i];
        const float4 pi = make_float4(a.x, a.y, a.z, a.w);
        fi = MULTI ? fid_of(vel[i]) : 0u;
        const float rho0 = C.fluids[fi].density0;
        const float umass = C.fluids[0].mass;
        Vel3 vi;
        if (UNI) {
            float2 b = D.vyz[i];
            vi = Vel3{a.w, b.x, b.y};
        } else {
            float4 s = D.vs[i];
            vi = Vel3{s.x, s.y, s.z};
        }
        float rho = 0.f, sq = 0.f, gx = 0.f, gy = 0.f, gz = 0.f, d = 0.f;
        const uint32_t n = fluid_stored(nf);
        const uint32_t nq = (n + 3u) >> 2;
        uint4 J = nq ? group(0u) : make_uint4(i, i, i, i);
        for (uint32_t q = 0; q < nq; ++q) {
            uint4 Jn = J;
            if (q + 1 < nq) Jn = group(q + 1);
            uint32_t j[4] = {J.x, J.y, J.z, J.w};
            float4 pj[4];
            Vel3 vj[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (q * 4u + u >= n) j[u] = i;  // tail slots of the last group: self (staged rows past n hold stale entries)
#pragma unroll
            for (int u = 0; u < 4; ++u) pj[u] = (UNI && (u & 1)) ? tex1Dfetch<float4>(D.tposrec, (int)j[u]) : __ldg(&D.posrec[j[u]]);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (UNI) {  // even contacts: (record via LSU, velocity via TEX), odd ones the other way round
                    float2 b = (u & 1) ? __ldg(&D.vyz[j[u]]) : tex1Dfetch<float2>(D.tvyz, (int)j[u]);
                    vj[u] = Vel3{pj[u].w, b.x, b.y};
                } else {
                    float4 s = tex1Dfetch<float4>(D.tvs, (int)j[u]);
                    vj[u] = Vel3{s.x, s.y, s.z};
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const bool ok = q * 4u + u < n;
                Pair p = make_pair<true, true>(pi, pj[u]);
                if (ok) {
                    const float mj = UNI ? umass : pj[u].w;
                    rho = fmaf(mj, p.w, rho);
                    float s = p.g * mj;  // m_j * gradient
                    float ax = s * p.dx, ay = s * p.dy, az = s * p.dz;
                    sq += ax * ax + ay * ay + az * az;
                    gx += ax; gy += ay; gz += az;
                    float dv = (vi.x - vj[u].x) * p.dx + (vi.y - vj[u].y) * p.dy + (vi.z - vj[u].z) * p.dz;
                    d = fmaf(dv * p.g, mj, d);
                }
            }
            J = Jn;
        }
        const uint32_t m = boundary_stored(nb);
        for (uint32_t k = 0; k < m; ++k) {
            const float4 pj = __ldg(&bpos[bentry(k)]);
            const Pair p = make_pair<true, true>(pi, pj);
            float mb = pj.w * rho0;  // boundary pseudo mass: vol_b * rho0_i
            rho = fmaf(mb, p.w, rho);
            float s = p.g * mb;
            float ax = s * p.dx, ay = s * p.dy, az = s * p.dz;
            sq += ax * ax + ay * ay + az * az;
            gx += ax; gy += ay; gz += az;
            float dv = vi.x * p.dx + vi.y * p.dy + vi.z * p.dz;  // boundary velocity ignored (dfsph_solver.rs:336-338)
            d = fmaf(dv * p.g, mb, d);
        }
        if (rho == 0.f) atomicOr(D.err, ERR_SEARCH_ZERO_DENSITY);  // assert!(!density.is_zero()) dfsph_solver.rs:662
        float den = sq + (gx * gx + gy * gy + gz * gz);
        float al = den <= 1.0e-5f ? 0.f : 1.0f / den;  // dfsph_solver.rs:209-213
        D.dens[i] = rho;
        D.alpha[i] = al;
        if (nf + nb < 20u) d = 0.f;  // min_neighbors_for_divergence_solve :62,301-314
        d = fmaxf(d, 0.f);
        D.divv[i] = d;
        if (UNI) D.pk4[i] = make_float4(a.x, a.y, a.z, d * al);
        else D.kappa[i] = d * al;
        e = d / rho0;
    }
    // The block's error partial, with block_sum's tree but no block barrier: the walks of a block's warps end at different
    // times, and a barrier made the finished warps wait for the slowest one (0.3-0.4 ms of the C3 search).  Each warp leaves
    // its sums in shared memory; the last warp to arrive adds them up.  read_error() sums the block partials.
    __shared__ float wsum[NBR_T / 32][MAX_FLUIDS];
    const uint32_t lane = threadIdx.x & 31u;
    const int nfl = MULTI ? C.n_fluids : 1;
    for (int f = 0; f < nfl; ++f) {
        const float s = warp_sum((valid && (!MULTI || fi == (uint32_t)f)) ? e : 0.f);
        if (lane == 0) wsum[threadIdx.x >> 5][f] = s;
    }
    uint32_t last = 0;
    if (lane == 0) {
        __threadfence_block();
        last = atomicAdd(&arrived, 1u) == NBR_T / 32 - 1;
    }
    if (__shfl_sync(0xffffffffu, last, 0)) {
        __threadfence_block();
        for (int f = 0; f < nfl; ++f) {
            const float s = warp_sum(lane < NBR_T / 32 ? *(volatile float*)&wsum[lane][f] : 0.f);
            if (lane == 0) D.partial[(size_t)blockIdx.x * nfl + f] = s;
        }
    }
}

// STAGE: the lists are staged per warp in shared memory and written out once the walk is done.  Storing each hit at its final
// place (((k >> 2) * stride + i) * 4 + (k & 3)) makes every 16-byte group of a list four partial writes spread over the whole
// kernel, with the lanes of a warp at different k: the sectors being filled (~29 MB at 10M particles) do not fit H100's L2.
// Staged, entry k of a lane is one STS at row k, column lane (bank-conflict-free whatever k each lane is at); the write-out
// then stores group g of 32 consecutive particles as 32 x 16 contiguous bytes, and boundary row k as 32 x 4.
// Entries past the staging rows go straight to their place in global memory, so any capacity works (list regrow
// included) while the shared-memory size stays fixed.  The row counts trade the share of staged entries against occupancy:
// 32 + 8 rows (20 KB per block) leave 10 blocks per SM, as many as the registers allow; at C3 (~33 contacts on average,
// up to ~51) 48 + 16 rows (6 blocks) made the search 26 % slower, 40 + 8 (9 blocks) 1 % slower (DESIGN.md §4a.11).
// Row order does not stage: the lanes of a warp are consecutive particles of one line and reach their k-th contact nearly
// together, so the per-hit stores already coalesce and staging only added cost (C2 rows: 0.300 vs 0.289 ms per search).
constexpr uint32_t NBR_SF = 32, NBR_SB = 8;  // staged fluid / boundary rows per lane (multiples of 4)

// The search shared by k_neighbors and k_neighbors_xy; `runs(pi, visit)` calls visit(lo, plane_start) for every z-run of cells the
// particle has to scan, lo being the cell id (cstart / bstart index) of the run's first cell; a run is always 3 cells.  The
// h-cell search visits the runs in sorted order and sets plane_start on the first run of each x-plane: it writes narrow lists
// unless out.wide (sph_lists.cuh), and raises maxcnt[2] if a window does not fit them.  Row order writes wide lists only.  STAGE (the
// h-cell search) also batches the candidate loads: both pay on h-cell runs only.  DENS: each particle then sweeps its own
// list with density_alpha_div, reading the staged entries from shared memory and the later ones back from global memory.
template <bool MULTI, bool STAGE, bool DENS, bool UNI, class Runs>
__device__ __forceinline__ void neighbor_lists(const float4* __restrict__ pos, const float4* __restrict__ vel, const uint32_t* __restrict__ cstart,
                                               const float4* __restrict__ bpos, const float4* __restrict__ bvel, const uint32_t* __restrict__ bstart,
                                               const ListsOut& out, uint32_t* __restrict__ maxcnt, const DensArgs& D, Runs runs) {
    __shared__ uint32_t stage[NBR_T / 32][NBR_SF + NBR_SB][32];
    __shared__ uint32_t arrived;  // DENS: warps of the block done with their density sweep
    if (DENS) {
        if (threadIdx.x == 0) arrived = 0;
        __syncthreads();  // (before the walk, while the block's warps are still together)
    }
    uint32_t(*const sf)[32] = stage[threadIdx.x >> 5];
    uint32_t(*const sb)[32] = sf + NBR_SF;
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nf = 0, nb = 0;
    // narrow lists (sph_lists.cuh; the h-cell search only): the first run of the x-plane being walked, and its window
    int lo_plane = 0;
    uint32_t plane = ~0u;
    Window win{};
    bool over = false;  // a window of this particle spans more than WINDOW_SLOTS slots
    const bool owned = i < C.n_owned;
    i += C.i_begin;
    if (owned) {
        const float4 pi = pos[i];
        const uint32_t fi = MULTI ? fid_of(vel[i]) : 0u;
        runs(pi, [&](int lo, bool plane_start) {
            if (STAGE && plane_start) {
                lo_plane = lo;
                ++plane;
            }
            scan_run<STAGE>(
                pi, pos, cstart[lo], cstart[lo + 3],
                [&](uint32_t j) {
                    if (!MULTI) return true;
                    uint32_t fj = fid_of(__ldg(&vel[j]));  // contacts.rs:355-362: different fluids need the groups test
                    return fi == fj || groups_test(C.fluids[fi].memberships, C.fluids[fi].filter, C.fluids[fj].memberships, C.fluids[fj].filter);
                },
                [&](uint32_t j) {
                    if (STAGE && nf < NBR_SF) sf[nf][lane] = j;
                    else out.fluid(i, nf, j, plane, out.wide ? 0u : cstart[lo_plane]);
                    ++nf;
                });
            if (C.n_bound)
                scan_run<STAGE>(
                    pi, bpos, bstart[lo], bstart[lo + 3],
                    [&](uint32_t j) {  // contacts.rs:347-352
                        uint32_t bj = fid_of(__ldg(&bvel[j]));
                        return groups_test(C.fluids[fi].memberships, C.fluids[fi].filter, C.bounds[bj].memberships, C.bounds[bj].filter);
                    },
                    [&](uint32_t j) {
                        if (STAGE && nb < NBR_SB) sb[nb][lane] = j;
                        else out.boundary(i, nb, j);
                        ++nb;
                    });
        });
        if (STAGE && NARROW_LISTS && !out.wide) {  // the windows: lo_plane is the first run of plane +1, planes are ny * nz cells apart
            const int P = C.ny * C.nz;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int lo = lo_plane - (2 - d) * P;
                win.base[d] = cstart[lo];
                over |= cstart[lo + 2 * C.nz + 3] - win.base[d] > WINDOW_SLOTS;
            }
            // lists that do not fit are redone wide; until then every entry decodes to a slot below WINDOW_SLOTS < n_fluid
            if (over) win = Window{};
            out.bases(i, win);
        }
        // write-out: the last group is padded; the capacities and NBR_SF are multiples of 4, so a staged group is whole
        if (STAGE) {
            const uint32_t sfn = min(fluid_stored(nf), NBR_SF);
            for (uint32_t k = 0; k < sfn; k += 4)
                out.group(i, k >> 2, make_uint4(sf[k][lane], sf[k + 1][lane], sf[k + 2][lane], sf[k + 3][lane]), nf, win);
            const uint32_t sbn = min(boundary_stored(nb), NBR_SB);
            for (uint32_t k = 0; k < sbn; ++k) out.boundary(i, k, sb[k][lane]);
        }
        out.pad(i, STAGE ? max(nf, NBR_SF) : nf, nf, win);  // pad the last group unless staged
        out.counts(i, nf, nb);
    }
    uint32_t mf = nf, mb = nb;
    for (int o = 16; o > 0; o >>= 1) {
        mf = max(mf, __shfl_xor_sync(0xffffffffu, mf, o));
        mb = max(mb, __shfl_xor_sync(0xffffffffu, mb, o));
    }
    const bool any_over = __any_sync(0xffffffffu, over);
    if (lane == 0) {
        if (mf) atomicMax(&maxcnt[0], mf);
        if (mb) atomicMax(&maxcnt[1], mb);
        if (any_over) atomicOr(&maxcnt[2], 1u);
    }
    if constexpr (DENS) {
        const Lists L = out.view();
        density_alpha_div<MULTI, UNI>(
            i, owned, nf, nb, vel, bpos, D, arrived,
            [&](uint32_t q) {
                const uint32_t k = q * 4u;
                if (STAGE && k < NBR_SF) return make_uint4(sf[k][lane], sf[k + 1][lane], sf[k + 2][lane], sf[k + 3][lane]);
                return out.group_ids(i, q);  // this thread's own stores above
            },
            [&](uint32_t k) { return STAGE && k < NBR_SB ? sb[k][lane] : L.boundary(i, k); });
    }
}

// DENS: DFSPH's density sweep runs in the search (density_alpha_div).  One fluid: 56 registers (9 blocks per SM).  Several
// fluids spill at 56 and get 64 (8 blocks); the generic solver kernels spill at 64 and are not bounded.
template <bool MULTI, bool DENS = false, bool UNI = false>
__global__ void __launch_bounds__(NBR_T, !DENS || SPH_GENERIC_KERNELS ? 1 : MULTI ? 8 : 9)
k_neighbors(const float4* __restrict__ pos, const float4* __restrict__ vel, const uint32_t* __restrict__ cstart,
            const float4* __restrict__ bpos, const float4* __restrict__ bvel, const uint32_t* __restrict__ bstart,
            ListsOut out, uint32_t* __restrict__ maxcnt /* StepScalars::max_nb */, DensArgs D) {
    neighbor_lists<MULTI, true, DENS, UNI>(pos, vel, cstart, bpos, bvel, bstart, out, maxcnt, D, [](const float4& pi, auto&& visit) {
        const int cx = cell_coord(pi.x), cy = cell_coord(pi.y), cz = cell_coord(pi.z);
        for (int ax = -1; ax <= 1; ++ax)
            for (int ay = -1; ay <= 1; ++ay) visit(cell_id(cx + ax, cy + ay, cz - 1), ay == -1);  // the z-run of cells cz-1..cz+1
    });
}

// Row order (Consts::xysub > 1): the same search over the bin rows within reach in x and y (5 x 5 rows of width h / 2 at xysub = 2
// instead of 3 x 3 of width h; arun() clips them to the reference's cells, so the contact sets are the reference's).  Neither
// staged nor batched: see scan_run and NBR_SF, so its density sweep reads the lists back from global memory.  No
// __launch_bounds__: with it ptxas holds the MULTI instantiation to 32 registers and spills.
template <bool MULTI, bool DENS = false, bool UNI = false>
__global__ void
k_neighbors_xy(const float4* __restrict__ pos, const float4* __restrict__ vel, const uint32_t* __restrict__ cstart,
               const float4* __restrict__ bpos, const float4* __restrict__ bvel, const uint32_t* __restrict__ bstart,
               ListsOut out, uint32_t* __restrict__ maxcnt /* StepScalars::max_nb */, DensArgs D) {
    neighbor_lists<MULTI, false, DENS, UNI>(pos, vel, cstart, bpos, bvel, bstart, out, maxcnt, D, [](const float4& pi, auto&& visit) {
        const int cx = cell_coord(pi.x), cy = cell_coord(pi.y), cz = cell_coord(pi.z);
        int xlo, xhi, ylo, yhi;
        arun(pi.x, cx, C.xysub, C.xysub_f, xlo, xhi);
        arun(pi.y, cy, C.xysub, C.xysub_f, ylo, yhi);
        for (int bx = xlo; bx <= xhi; ++bx)
            for (int by = ylo; by <= yhi; ++by) visit(cell_id(bx, by, cz - 1), false);
    });
}
// boundary volumes in row order: every bin of the 3 x 3 x 3 reference cells around the particle
__global__ void __launch_bounds__(128)
k_boundary_volumes_xy(const float4* __restrict__ bpos, const float4* __restrict__ bvel, const uint32_t* __restrict__ bstart, float* __restrict__ bvol,
                      unsigned long long* __restrict__ ncontacts, int* __restrict__ err) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t cnt = 0;
    if (i < C.n_bound) {
        float4 pi = bpos[i];
        uint32_t bi = fid_of(bvel[i]);
        const int cx = cell_coord(pi.x), cy = cell_coord(pi.y), cz = cell_coord(pi.z);
        float den = 0.f;
        for (int bx = (cx - 1) * C.xysub; bx < (cx + 2) * C.xysub; ++bx)
            for (int by = (cy - 1) * C.xysub; by < (cy + 2) * C.xysub; ++by) {
                const int base = cell_id(bx, by, cz - 1);
                const uint32_t s = bstart[base], e = bstart[base + 3];
                for (uint32_t j = s; j < e; ++j) {
                    float4 pj = __ldg(&bpos[j]);
                    float dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
                    float d2 = dist2_exact(dx, dy, dz);
                    if (d2 <= C.h2) {
                        uint32_t bj = fid_of(__ldg(&bvel[j]));
                        if (bi == bj || groups_test(C.bounds[bi].memberships, C.bounds[bi].filter, C.bounds[bj].memberships, C.bounds[bj].filter)) {
                            den += C.kgen ? kernel_w_kind(C.kw, __fsqrt_rn(d2)) : kernel_w(sqrtf(d2));
                            ++cnt;
                        }
                    }
                }
            }
        if (den == 0.f) atomicOr(err, ERR_ZERO_DENSITY);
        bvol[i] = 1.0f / den;
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(ncontacts, (unsigned long long)cnt);
}

// a4: compute_boundary_volumes dfsph_solver.rs:72-96 — vol_b = 1 / sum_{b'} W_bb' over boundary-boundary
// contacts (same boundary, or other boundaries passing the groups test; self included).
__global__ void __launch_bounds__(128)
k_boundary_volumes(const float4* __restrict__ bpos, const float4* __restrict__ bvel, const uint32_t* __restrict__ bstart, float* __restrict__ bvol,
                   unsigned long long* __restrict__ ncontacts, int* __restrict__ err) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t cnt = 0;
    if (i < C.n_bound) {
        float4 pi = bpos[i];
        uint32_t bi = fid_of(bvel[i]);
        int cx = cell_coord(pi.x), cy = cell_coord(pi.y), cz = cell_coord(pi.z);
        float den = 0.f;
        for (int ax = -1; ax <= 1; ++ax)
            for (int ay = -1; ay <= 1; ++ay) {
                int base = cell_id(cx + ax, cy + ay, cz - 1);  // the three cells cz-1..cz+1
                uint32_t s = bstart[base], e = bstart[base + 3];
                for (uint32_t j = s; j < e; ++j) {
                    float4 pj = __ldg(&bpos[j]);
                    float dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
                    float d2 = dist2_exact(dx, dy, dz);
                    if (d2 <= C.h2) {
                        uint32_t bj = fid_of(__ldg(&bvel[j]));
                        if (bi == bj || groups_test(C.bounds[bi].memberships, C.bounds[bi].filter, C.bounds[bj].memberships, C.bounds[bj].filter)) {
                            den += C.kgen ? kernel_w_kind(C.kw, __fsqrt_rn(d2)) : kernel_w(sqrtf(d2));
                            ++cnt;
                        }
                    }
                }
            }
        if (den == 0.f) atomicOr(err, ERR_ZERO_DENSITY);  // assert!(!denominator.is_zero()) dfsph_solver.rs:92
        bvol[i] = 1.0f / den;
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(ncontacts, (unsigned long long)cnt);
}
__global__ void k_set_w(uint32_t n, float4* __restrict__ a, const float* __restrict__ w) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i].w = w[i];
}

// ------------------------------------------------------------------------------------------------
// Error reduction + elementwise (streaming) kernels.  The neighbour-gather passes live in sph_passes.cuh.
// ------------------------------------------------------------------------------------------------
// One block per fluid: fixed-order sum of the per-block partials.
__global__ void k_reduce_partials(const float* __restrict__ partial, uint32_t nblocks, int n_fluids, float* __restrict__ out) {
    __shared__ float sm[32];
    int f = blockIdx.x;
    float s = 0.f;
    for (uint32_t b = threadIdx.x; b < nblocks; b += blockDim.x) s += partial[(size_t)b * n_fluids + f];
    s = block_sum(s, sm);
    if (threadIdx.x == 0) out[f] = s;
}

#ifndef SPH_PASS_T
#define SPH_PASS_T 128
#endif
#ifndef SPH_PASS_MINB
#define SPH_PASS_MINB 9   // Jacobi-loop / density kernels: 56 registers, 9 blocks of 128 per SM
#endif
#ifndef SPH_FORCE_MINB
#define SPH_FORCE_MINB 8  // force kernels gather more per contact: 64 registers avoid spills
#endif
constexpr int PASS_T = SPH_PASS_T;  // threads per block of the gather passes

// Where v* lives, as the streaming passes see it (VStarRecords on the host): on the uniform-mass path (pvx != nullptr) only in
// the packed records pvx.w and vyz, and vs is not written; else in vs.  The passes take it as a __grid_constant__ parameter
// and read its pointers from the parameter bank, as they would plain pointer parameters.
struct VStar {
    float4* vs;
    float4* pvx;
    float2* vyz;
    // for passes that do not write v*: reads through the read-only data cache
    __device__ __forceinline__ float4 load(uint32_t i) const {
        if (!pvx) return __ldg(&vs[i]);
        const float2 b = __ldg(&vyz[i]);
        return make_float4(__ldg(&pvx[i].w), b.x, b.y, 0.f);
    }
    // v* of slot i, and (packed) the position p that shares its record
    __device__ __forceinline__ void store(uint32_t i, const float4& p, float sx, float sy, float sz) const {
        if (pvx) {
            pvx[i] = make_float4(p.x, p.y, p.z, sx);
            vyz[i] = make_float2(sy, sz);
        } else {
            vs[i] = make_float4(sx, sy, sz, 0.f);
        }
    }
};

// The fluid reorder fused with v* = vel + vc: the sorted pos / vel / vc are in registers anyway, so v* and the packed
// gather records are written by the same pass (saves re-reading 48 B per particle and a launch).  g.in4 / out4 [0..2] = pos, vel, vc.
__global__ void k_gather_vstar(uint32_t n, const uint32_t* __restrict__ perm, GatherSet g, const __grid_constant__ VStar vst) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t src = perm[s];
    const float4 p = g.in4[0][src], v = g.in4[1][src], c = g.in4[2][src];
    g.out4[0][s] = p;
    g.out4[1][s] = v;
    g.out4[2][s] = c;
#pragma unroll
    for (int a = 0; a < 4; ++a)
        if (a < g.n1) g.out1[a][s] = g.in1[a][src];
    vst.store(s, p, v.x + c.x, v.y + c.y, v.z + c.z);
}

// a10: update_velocities dfsph_solver.rs:422-430 + zero vc :689-691 + acc = gravity (predict_advection :574-578).
// vel += vc is written as vel = v*: v* was materialised as vel + vc by the producer, so the result is bitwise the
// same for owned particles, and ghost particles (multi-GPU) only carry an up-to-date v*.
// xs (optional): a force sum of the divergence loop (k_vel_divergence_xsph_u): acc = g + xs * scale, rounded like the force
// pass's `acc += f * scale` on top of the gravity written here.  XSPH sums: scale = inv_dt; the Akinci force: scale = 1, so
// acc = g + f exactly as `acc = g; acc += f`.
__global__ void k_fold_velocities(float4* __restrict__ vel, float4* __restrict__ vc, const __grid_constant__ VStar vst, float4* __restrict__ acc, float gx, float gy,
                                  float gz, const float4* __restrict__ xs, float scale) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.n_fluid) return;
    const float4 v = vel[i], s = vst.load(i);
    vel[i] = make_float4(s.x, s.y, s.z, v.w);
    vc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    float ax = gx, ay = gy, az = gz;
    if (xs) {
        float4 f = xs[i];
        ax = __fadd_rn(gx, __fmul_rn(f.x, scale));
        ay = __fadd_rn(gy, __fmul_rn(f.y, scale));
        az = __fadd_rn(gz, __fmul_rn(f.z, scale));
    }
    acc[i] = make_float4(ax, ay, az, 0.f);
}
// update_velocities + the gravity / folded-force acceleration + integrate_and_clear_accelerations in ONE pass, for steps whose force
// phase launches nothing (no plugin, or only the force whose sum rode with the divergence loop): same arithmetic, in the same
// order, as k_fold_velocities followed by k_integrate_acc.  Ghost slots (multi-GPU) only take the fold part.
// Uniform mass (vst.pvx != nullptr): the whole of pvx[i] is loaded anyway, so it is stored whole (xyz unchanged) rather than
// as a partial .w store.
__global__ void k_fold_integrate(float4* __restrict__ vel, float4* __restrict__ vc, const __grid_constant__ VStar vst, float4* __restrict__ acc, float gx, float gy,
                                 float gz, const float4* __restrict__ xs, float scale, float dt_new) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= C.n_fluid) return;
    float4 *const vs = vst.vs, *const pvx = vst.pvx;
    float2* const vyz = vst.vyz;
    const float4 v = vel[i];
    float4 s, r;  // v*, and (uniform mass) the packed record
    if (pvx) {
        r = pvx[i];
        const float2 b = vyz[i];
        s = make_float4(r.w, b.x, b.y, 0.f);
    } else {
        s = vs[i];
    }
    const float4 nv = make_float4(s.x, s.y, s.z, v.w);
    vel[i] = nv;
    const bool owned = i >= C.i_begin && i < C.i_begin + C.n_owned;
    float ax = gx, ay = gy, az = gz;
    if (xs) {
        const float4 f = xs[i];
        ax = __fadd_rn(gx, __fmul_rn(f.x, scale));
        ay = __fadd_rn(gy, __fmul_rn(f.y, scale));
        az = __fadd_rn(gz, __fmul_rn(f.z, scale));
    }
    acc[i] = make_float4(ax, ay, az, 0.f);
    if (!owned) {
        vc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    const float cx = __fmul_rn(ax, dt_new), cy = __fmul_rn(ay, dt_new), cz = __fmul_rn(az, dt_new);  // vc = 0 + acc * dt
    vc[i] = make_float4(cx, cy, cz, 0.f);
    const float sx = nv.x + cx, sy = nv.y + cy, sz = nv.z + cz;
    if (pvx) {
        pvx[i] = make_float4(r.x, r.y, r.z, sx);
        vyz[i] = make_float2(sy, sz);
    } else {
        vs[i] = make_float4(sx, sy, sz, 0.f);
    }
}
// IISPH variant: accelerations += gravity only (vc is already zero, velocities untouched).
__global__ void k_set_gravity(const float4* __restrict__ vel, float4* __restrict__ vs, float4* __restrict__ acc, float gx, float gy, float gz) {
    SPH_OWNED_INDEX(i)
    float4 v = vel[i];
    vs[i] = make_float4(v.x, v.y, v.z, 0.f);
    acc[i] = make_float4(gx, gy, gz, 0.f);
}

// a18: integrate_and_clear_accelerations dfsph_solver.rs:505-518 (+ v* = vel + vc).  The accelerations are NOT cleared here:
// the next step's k_fold_velocities / k_set_gravity overwrites them with gravity before any force adds to them, so the
// array doubles as the SPH_DBG_ACCELERATION view and the pass saves 32 B per particle of stores.
__global__ void k_integrate_acc(const float4* __restrict__ vel, float4* __restrict__ vc, const __grid_constant__ VStar vst, const float4* __restrict__ acc, float dt) {
    SPH_OWNED_INDEX(i)
    float4 a = acc[i], c = vc[i], v = vel[i];
    c.x += a.x * dt; c.y += a.y * dt; c.z += a.z * dt;
    vc[i] = c;
    float sx = v.x + c.x, sy = v.y + c.y, sz = v.z + c.z;
    if (vst.pvx) {  // uniform mass: v* only in the packed records
        vst.pvx[i].w = sx;  // xyz already hold the position
        vst.vyz[i] = make_float2(sy, sz);
    } else {
        vst.vs[i] = make_float4(sx, sy, sz, 0.f);
    }
}

// The CFL bound's reduction (TimestepManager::max_substep timestep_manager.rs:36-46): max over the owned fluid particles of
// |v + a * remaining|^2, in the reference's operation order (v + a * R, then ((x^2 + y^2) + z^2)).  Non-negative floats
// order like their bit patterns, so each warp reduces the bits with __reduce_max_sync and one lane atomicMax-es them into
// *out, which the host zeroes per substep: the result does not depend on the block order.  A NaN (bits above +inf's)
// wins the reduction, and the host then takes the largest substep count.
__global__ void k_cfl_max(const float4* __restrict__ vel, const float4* __restrict__ acc, float remaining, unsigned int* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned int bits = 0u;
    if (i < C.n_owned) {
        const float4 v = vel[C.i_begin + i], a = acc[C.i_begin + i];
        const float x = __fadd_rn(v.x, __fmul_rn(a.x, remaining));
        const float y = __fadd_rn(v.y, __fmul_rn(a.y, remaining));
        const float z = __fadd_rn(v.z, __fmul_rn(a.z, remaining));
        bits = __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    }
    bits = __reduce_max_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31u) == 0u && bits) atomicMax(out, bits);
}

// a22: update_positions dfsph_solver.rs:411-420: pos += (vel + vc) * dt.  bounds_out (optional): the cell-coordinate AABB of
// the NEW positions (what k_bounds computes), so the next step's grid is sized without a bounds pass and its host round trip.
__global__ void k_update_positions(float4* __restrict__ pos, const __grid_constant__ VStar vst, float dt, CellBox* __restrict__ bounds_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < C.n_owned;
    i += C.i_begin;
    CellBox b = CELL_BOX_EMPTY;
    if (valid) {
        float4 p = pos[i];
        const float4 v = vst.load(i);
        p.x += v.x * dt; p.y += v.y * dt; p.z += v.z * dt;
        pos[i] = p;
        if (bounds_out) cell_box_add(b, p.x, p.y, p.z, C.h);
    }
    if (!bounds_out) return;
    cell_box_commit_block(b, bounds_out);
}

__device__ __forceinline__ float powi3(float x) { return x * x * x; }
// akinci2013_surface_tension.rs:71-88
__device__ __forceinline__ float cohesion_kernel(float r, float coh_norm, float h6_64) {
    float hr = powi3(C.h - r) * powi3(r);
    float c = r <= C.h * 0.5f ? 2.0f * hr - h6_64 : (r <= C.h ? hr : 0.f);
    return coh_norm * c;
}

// akinci2013_surface_tension.rs:90-111
__device__ __forceinline__ float adhesion_kernel(float r, float adh_norm) {
    if (r > C.h * 0.5f && r <= C.h) {
        float x = fmaxf(-4.0f * r * r / C.h + 6.0f * r - 2.0f * C.h, 0.f);
        return adh_norm * sqrtf(sqrtf(x));  // powf(0.25)
    }
    return 0.f;
}

__global__ void k_iota(uint32_t n, uint32_t* __restrict__ a) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) a[s] = s;
}
// ------------------------------------------------------------------------------------------------
// Slab decomposition helpers (sph_slab.inl): classification by cell column, stream compaction.
// ------------------------------------------------------------------------------------------------
// Owned slots [ob, ob + on) are classified by their CURRENT cell column in ONE pass.  Nothing is compacted: particles that
// left the slab are only flagged `dead` (the counting sort that follows drops them), and the few particles the neighbours
// need — emigrants and the kept particles of my two boundary columns — are appended to small staging buffers with one
// atomic per warp.  Their order inside the buffers is arbitrary; the receiver's sort orders every cell by particle id.
// counts[1..5] = #left, #right, #col-left, #col-right, #particles that jumped > 1 column.
struct SlabOut {  // staging arrays of k_slab_classify
    float4 *pos, *vel, *vc;
    uint32_t* gid;
};
__device__ __forceinline__ uint32_t warp_append(bool pred, uint32_t* counter) {
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (!m) return 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, leader = __ffs((int)m) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(counter, (uint32_t)__popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    return pred ? base + (uint32_t)__popc(m & ((1u << lane) - 1u)) : 0xFFFFFFFFu;
}
__global__ void k_slab_classify(const float4* __restrict__ pos, const float4* __restrict__ vel, const float4* __restrict__ vc, const uint32_t* __restrict__ gid,
                                uint32_t ob, uint32_t on, int lo, int hi, int has_left, int has_right, uint32_t* __restrict__ dead, SlabOut out_l, SlabOut out_r,
                                SlabOut col_l, SlabOut col_r, uint32_t cap_out, uint32_t cap_col, uint32_t* __restrict__ counts) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = t < on;
    const uint32_t s = ob + (in ? t : 0u);
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
    bool left = false, right = false, cl = false, cr = false, jumped = false;
    if (in) {
        p = pos[s];
        const int cx = cell_coord(p.x);
        left = has_left && cx < lo;
        right = has_right && cx >= hi;
        cl = !left && !right && has_left && cx == lo;
        cr = !left && !right && has_right && cx == hi - 1;
        jumped = (left && cx < lo - 1) || (right && cx > hi);
        dead[t] = (left || right) ? 1u : 0u;
    }
    const uint32_t kl = warp_append(left, &counts[1]), kr = warp_append(right, &counts[2]);
    const uint32_t kcl = warp_append(cl, &counts[3]), kcr = warp_append(cr, &counts[4]);
    warp_append(jumped, &counts[5]);
    if (!(left || right || cl || cr)) return;
    const float4 v = vel[s], c = vc[s];
    const uint32_t g = gid[s];
    if (left && kl < cap_out) { out_l.pos[kl] = p; out_l.vel[kl] = v; out_l.vc[kl] = c; out_l.gid[kl] = g; }
    if (right && kr < cap_out) { out_r.pos[kr] = p; out_r.vel[kr] = v; out_r.vc[kr] = c; out_r.gid[kr] = g; }
    if (cl && kcl < cap_col) { col_l.pos[kcl] = p; col_l.vel[kcl] = v; col_l.vc[kcl] = c; col_l.gid[kcl] = g; }
    if (cr && kcr < cap_col) { col_r.pos[kcr] = p; col_r.vel[kcr] = v; col_r.vc[kcr] = c; col_r.gid[kcr] = g; }
}
// counts[8..9] = {#emigrants left, #col-left}, counts[10..11] = {#emigrants right, #col-right}: the two 8-byte messages
__global__ void k_slab_pack_counts(uint32_t* __restrict__ counts) {
    if (threadIdx.x == 0) {
        counts[8] = counts[1]; counts[9] = counts[3];
        counts[10] = counts[2]; counts[11] = counts[4];
    }
}
__global__ void k_iota_from(uint32_t n, uint32_t start, uint32_t* __restrict__ a) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) a[s] = start + s;
}

// ------------------------------------------------------------------------------------------------
// Ghost exchange over NVLink peer memory (sph_slab.inl).  Every rank maps its two neighbours' landing zones ("boxes",
// cudaIpc) and the producer side WRITES its boundary columns straight into the neighbour's box with plain st.global
// over NVLink, then publishes a sequence number (release, system scope); the consumer side spins on its own flag
// (acquire, system scope) and copies box -> ghost slots.  No NCCL, no host involvement, ~10 us per exchange.
// ------------------------------------------------------------------------------------------------
struct P2PSeg {           // one contiguous array range travelling in a message
    const char* src;      // sender: local source; receiver: unused
    char* dst;            // receiver: local ghost range; sender: unused
    uint32_t box_off;     // byte offset inside the box (16-byte aligned)
    uint32_t bytes;       // multiple of 4
};
struct P2PMsg {           // one direction (to / from one neighbour)
    char* box;            // sender: the NEIGHBOUR's box (peer pointer); receiver: my own box
    uint32_t* flag;       // sender: the neighbour's flag (peer pointer); receiver: my own flag
    P2PSeg seg[4];
    int n_seg;
    uint32_t total_words;  // sum of bytes / 4
};
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
// bounded spin (a peer that never arrives must not hang the GPU): ~2 s of SM clock, then the (sticky) error flag
__device__ __forceinline__ bool p2p_wait(const uint32_t* flag, uint32_t seq, int* err) {
    if (*reinterpret_cast<volatile int*>(err) & ERR_PEER_TIMEOUT) return false;  // an earlier exchange of this step already timed out: do not wait again
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(flag) - seq) < 0) {
        if (clock64() - t0 > 4000000000LL) {
            atomicOr(err, ERR_PEER_TIMEOUT);
            return false;
        }
        __nanosleep(64);
    }
    return true;
}
// blockIdx.y = direction (0: left neighbour, 1: right neighbour)
__global__ void k_p2p_push(P2PMsg m0, P2PMsg m1, uint32_t seq0, uint32_t seq1, uint32_t* __restrict__ tickets) {
    const P2PMsg& m = blockIdx.y ? m1 : m0;
    if (!m.box) return;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (int s = 0; s < m.n_seg; ++s) {
        const uint32_t* __restrict__ src = reinterpret_cast<const uint32_t*>(m.seg[s].src);
        uint32_t* dst = reinterpret_cast<uint32_t*>(m.box + m.seg[s].box_off);
        const uint32_t nw = m.seg[s].bytes >> 2;
        const uint32_t n4 = nw >> 2;  // ranges start 16-byte aligned on both sides whenever the element size is a multiple of 16
        if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
            const uint4* s4 = reinterpret_cast<const uint4*>(src);
            uint4* d4 = reinterpret_cast<uint4*>(dst);
            for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n4; k += stride) d4[k] = s4[k];
            for (uint32_t k = 4 * n4 + blockIdx.x * blockDim.x + threadIdx.x; k < nw; k += stride) dst[k] = src[k];
        } else {
            for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nw; k += stride) dst[k] = src[k];
        }
    }
    __threadfence_system();
    __shared__ bool last;
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(&tickets[blockIdx.y], 1u) == gridDim.x - 1;
    __syncthreads();
    if (last && threadIdx.x == 0) {
        tickets[blockIdx.y] = 0;
        __threadfence_system();
        st_release_sys(m.flag, blockIdx.y ? seq1 : seq0);
    }
}
__global__ void k_p2p_pull(P2PMsg m0, P2PMsg m1, uint32_t seq0, uint32_t seq1, int* __restrict__ err) {
    const P2PMsg& m = blockIdx.y ? m1 : m0;
    if (!m.box) return;
    __shared__ bool ok;
    if (threadIdx.x == 0) ok = p2p_wait(m.flag, blockIdx.y ? seq1 : seq0, err);
    __syncthreads();
    if (!ok) return;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (int s = 0; s < m.n_seg; ++s) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(m.box + m.seg[s].box_off);
        uint32_t* dst = reinterpret_cast<uint32_t*>(m.seg[s].dst);
        const uint32_t nw = m.seg[s].bytes >> 2;
        const uint32_t n4 = nw >> 2;
        if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
            const uint4* s4 = reinterpret_cast<const uint4*>(src);
            uint4* d4 = reinterpret_cast<uint4*>(dst);
            for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n4; k += stride) d4[k] = __ldcv(&s4[k]);  // written by a peer: bypass L1
            for (uint32_t k = 4 * n4 + blockIdx.x * blockDim.x + threadIdx.x; k < nw; k += stride) dst[k] = __ldcv(&src[k]);
        } else {
            for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nw; k += stride) dst[k] = __ldcv(&src[k]);
        }
    }
}
// All-ranks sum of a few floats (Jacobi error means) through peer memory: rank r writes its values into slot r of EVERY
// rank's table, publishes, waits for all slots and sums them in rank order (deterministic, same result on every rank).
struct P2PPeers {
    float* red[8];         // red[p]: rank p's table  [buf][rank][MAX_FLUIDS]
    uint32_t* red_flag[8]; // rank p's flags          [buf][rank]
};
__global__ void k_p2p_allreduce(float* __restrict__ vals, int n, int rank, int nranks, P2PPeers P, uint32_t seq, int* __restrict__ err) {
    const int buf = (int)(seq & 1u);
    const int t = threadIdx.x;
    // thread (p, f): write vals[f] into rank p's table
    for (int k = t; k < nranks * n; k += blockDim.x) {
        const int p = k / n, f = k % n;
        P.red[p][((size_t)buf * 8 + rank) * MAX_FLUIDS + f] = vals[f];
    }
    __threadfence_system();
    __syncthreads();
    for (int p = t; p < nranks; p += blockDim.x) st_release_sys(&P.red_flag[p][buf * 8 + rank], seq);
    __shared__ int ok;
    if (t == 0) ok = 1;
    __syncthreads();
    for (int p = t; p < nranks; p += blockDim.x)
        if (!p2p_wait(&P.red_flag[rank][buf * 8 + p], seq, err)) ok = 0;
    __syncthreads();
    if (!ok) return;
    for (int f = t; f < n; f += blockDim.x) {
        float s = 0.f;
        for (int p = 0; p < nranks; ++p) s += __ldcv(&P.red[rank][((size_t)buf * 8 + p) * MAX_FLUIDS + f]);
        vals[f] = s;
    }
}

// ------------------------------------------------------------------------------------------------
// ParticlesContacts materialisation for host NonPressureForce plugins (nonpressure_force.rs:15-27 hands
// `fluid_fluid_contacts` / `fluid_boundaries_contacts` to solve(); Contact = {i_model, j_model, i, j, weight, gradient},
// contacts.rs:12-27).  CSR in ORIGINAL particle order; entries of a particle keep the list order (ascending sorted j).
// ------------------------------------------------------------------------------------------------
struct OffsetTable {
    uint32_t off[MAX_FLUIDS > MAX_BOUNDARIES ? MAX_FLUIDS + 1 : MAX_BOUNDARIES + 1];
};
__global__ void k_contacts_count(uint32_t n, const uint32_t* __restrict__ orig, const uint32_t* __restrict__ cnt, uint32_t cap, uint32_t* __restrict__ out) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) out[orig[s]] = min(cnt[s], cap);
}
// one thread per sorted slot: writes its particle's contacts at scan[orig[s]]..
template <bool BOUNDARY>
__global__ void k_contacts_fill(uint32_t n, const float4* __restrict__ pos, const float4* __restrict__ other_pos, const float4* __restrict__ other_vel,
                                const uint32_t* __restrict__ orig, const uint32_t* __restrict__ other_orig, Lists L,
                                const uint32_t* __restrict__ scan, OffsetTable tab, uint32_t* __restrict__ out_j,
                                uint32_t* __restrict__ out_model, float* __restrict__ out_w, float* __restrict__ out_g) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t i = s + C.i_begin;
    const float4 pi = pos[i];
    const uint32_t m = BOUNDARY ? L.boundary_count(i) : L.fluid_count(i);
    size_t base = scan[orig[i]];
    for (uint32_t k = 0; k < m; ++k) {
        const uint32_t j = BOUNDARY ? L.boundary(i, k) : L.fluid(i, k);
        const float4 pj = other_pos[j];
        const Pair p = make_pair<true, true>(pi, pj);
        const uint32_t model = fid_of(other_vel[j]);
        out_j[base + k] = other_orig[j] - tab.off[model];
        out_model[base + k] = model;
        out_w[base + k] = p.w;
        out_g[3 * (base + k) + 0] = p.g * p.dx;
        out_g[3 * (base + k) + 1] = p.g * p.dy;
        out_g[3 * (base + k) + 2] = p.g * p.dz;
    }
}

__global__ void k_sum_u32(uint32_t n, const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, unsigned long long* __restrict__ out) {
    unsigned long long s = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) s += (unsigned long long)a[i] + b[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// ------------------------------------------------------------------------------------------------
// Jacobi-loop exits (dfsph_solver.rs:153-158, :347-352, :450, :486), shared by the host loops and the device decisions of
// the step graph (sph_graph.inl), so that both end a loop after the same evaluation.
// ------------------------------------------------------------------------------------------------
// The largest per-fluid mean sums[f] / n[f] over the fluids with n[f] > 0 (n as float, from the particle count); 0 without
// any, and a NaN mean never wins (the comparison of std::max).
__host__ __device__ inline float loop_error(const float* sums, const float* n, int nf) {
    float mx = 0.f;
    for (int f = 0; f < nf; ++f)
        if (n[f] > 0.f) {
            const float e = sums[f] / n[f];
            mx = mx < e ? e : mx;
        }
    return mx;
}
// Whether the loop breaks after evaluation i with error avg: the divergence bound is max_error * inv_dt * 0.01 (products only, so
// nothing contracts into an FMA), the density bound max_error itself.
__host__ __device__ inline bool loop_exit(float avg, float max_error, bool divergence, float inv_dt, uint32_t i, uint32_t min_iter) {
    const float max_err = divergence ? max_error * inv_dt * 0.01f : max_error;
    return avg <= max_err && i >= min_iter;
}
// One Jacobi loop: maxit evaluations at most (DFSPH: force + 1 when force >= 0), the exit rule, the fluid sizes.
struct LoopRule {
    uint32_t maxit, min_iter;
    int32_t force;
    float max_error, inv_dt;
    int divergence, nf;
    float n[MAX_FLUIDS];
};
// The decision after evaluation i of loop r: whether its error is read (error() is called then and only then), whether the
// loop breaks, and whether another evaluation follows.  A pinned count (force >= 0) reads nothing and breaks at i == force.
// The break needs i >= min_iter (dfsph_solver.rs:450, :486), so an earlier evaluation that is not the last cannot end the
// loop and the next one reports a fresher error: it reads nothing, which spares the host a read-back.
struct LoopDecision {
    bool read, brk, more;
};
#pragma nv_exec_check_disable  // error() is a host lambda on the host (read_error) and a device lambda in k_loop_decide
template <class Error>
__host__ __device__ inline LoopDecision loop_decision(const LoopRule& r, uint32_t i, Error error) {
    LoopDecision d;
    d.read = r.force < 0 && !(i < r.min_iter && i + 1 < r.maxit);
    d.brk = r.force >= 0 ? (int)i >= r.force : d.read && loop_exit(error(), r.max_error, r.divergence != 0, r.inv_dt, i, r.min_iter);
    d.more = !d.brk && i + 1 < r.maxit;
    return d;
}

// Which fused sums are valid when the divergence loop ends, from its counts (xsf: xsph_fusable, akf: akinci_fusable_u).  The
// loop's update 0 carries the Akinci normals (an update ran), its evaluation 1 the Akinci force (two evaluations ran); the
// XSPH sums of an evaluation i >= 1 are valid when the loop ended on that evaluation (one update fewer than evaluations).
enum : uint32_t { FOLD_XS = 1, FOLD_NR4 = 2, FOLD_AKINCI = 4 };
__host__ __device__ inline uint32_t fold_state(bool xsf, bool akf, uint32_t n_eval, uint32_t n_iter) {
    const uint32_t xs = xsf && n_eval >= 2 && n_iter + 1 == n_eval;
    const uint32_t nr4 = akf && n_iter >= 1, ak = akf && n_eval >= 2;
    return xs * FOLD_XS | nr4 * FOLD_NR4 | ak * FOLD_AKINCI;
}

// ---- step graph (sph_world_step_many, sph_graph.inl): device-side control ------------------------------------------------
// One record per step of a call; the layout of sph_step_record.
struct StepRec {
    uint32_t n_div_iter, n_press_iter, n_div_eval, n_press_eval;
    float last_div_err, last_dens_err;
    uint32_t max_neighbors, on_device;
    unsigned long long n_contacts;
};
enum { GRAPH_STOP_NONE = 0, GRAPH_STOP_REDO = 1, GRAPH_STOP_LEFT = 2, GRAPH_STOP_ERROR = 3 };
// What the graph carries from kernel to kernel.  REDO: the step found lists longer than their capacity and stopped after its
// sort; LEFT: the step's new positions left the grid envelope or are not finite; ERROR: the step raised the error flag.
struct GraphCtl {
    uint32_t left;  // steps still to run
    uint32_t step;  // steps completed (index of the running step's record)
    uint32_t stop;  // GRAPH_STOP_*
    uint32_t it;    // iteration of the running Jacobi loop
};
// Conditional handles a decision sets: [0] to "an update follows", [1] to "an update and another evaluation follow",
// [2] to "an update follows and ends the loop", [3] and [4] to 0 (unused entries are 0 and not set).  k_fold_arm: [s] to
// "the loop ended in state s".
struct Decide {
    cudaGraphConditionalHandle h[8];
};

__global__ void k_graph_arm(const GraphCtl* ctl, cudaGraphConditionalHandle h) {
    cudaGraphSetConditional(h, (ctl->stop == GRAPH_STOP_NONE && ctl->left > 0) ? 1u : 0u);
}

// After evaluation i (i0 >= 0: this i, else the running loop's next) of a loop: loop_decision with its counts and error
// read, and the handles of what follows.
__global__ void k_loop_decide(GraphCtl* ctl, StepRec* rec, const float* loop_err, LoopRule r, int i0, Decide d) {
    const uint32_t i = i0 >= 0 ? (uint32_t)i0 : ctl->it + 1;
    ctl->it = i;
    StepRec& R = rec[ctl->step];
    (r.divergence ? R.n_div_eval : R.n_press_eval)++;
    const LoopDecision x = loop_decision(r, i, [&] {
        const float avg = loop_error(loop_err, r.n, r.nf);
        (r.divergence ? R.last_div_err : R.last_dens_err) = avg;
        return avg;
    });
    if (!x.brk) (r.divergence ? R.n_div_iter : R.n_press_iter)++;
    const unsigned v[5] = {!x.brk, x.more, !x.brk && !x.more, 0u, 0u};
    for (int k = 0; k < 5; ++k)
        if (d.h[k]) cudaGraphSetConditional(d.h[k], v[k]);
}

// After the divergence loop: h[s] is the post-loop branch of fold state s, set from the step's counts
__global__ void k_fold_arm(const GraphCtl* ctl, const StepRec* rec, int xsf, int akf, Decide d) {
    const StepRec& R = rec[ctl->step];
    const uint32_t s = fold_state(xsf, akf, R.n_div_eval, R.n_div_iter);
    for (uint32_t k = 0; k < 8; ++k)
        if (d.h[k]) cudaGraphSetConditional(d.h[k], k == s ? 1u : 0u);
}

// After the neighbour search of a graph step: the list capacity and width checks and error word of phase_neighbors' read-back.
// A list longer than its capacity, narrow lists a window does not fit (or a boundary-volume error) stop the graph before the
// solver; the host redoes the step.
__global__ void k_lists_check(GraphCtl* ctl, StepRec* rec, const StepScalars* ss, uint32_t cap_f, uint32_t cap_b, cudaGraphConditionalHandle h) {
    const uint32_t mf = ss->max_nb[0], mb = ss->max_nb[1];
    const bool ok = !(ss->err & ~ERR_SEARCH_ZERO_DENSITY) && mf <= cap_f && mb <= cap_b && !ss->max_nb[2];
    rec[ctl->step].max_neighbors = mf;
    if (!ok) ctl->stop = GRAPH_STOP_REDO;
    cudaGraphSetConditional(h, ok ? 1u : 0u);
}

// Initial value of k_update_positions' bounds
__global__ void k_bounds_init(CellBox* b) { *b = CELL_BOX_EMPTY; }

// End of a graph step: the record's contacts, the count, and the stops of world_substep's read-back: the error word, and new
// positions outside the envelope env (the bad flag unused) or not finite.
__global__ void k_step_end(GraphCtl* ctl, StepRec* rec, const StepScalars* ss, CellBox env, unsigned long long bb_contacts) {
    StepRec& R = rec[ctl->step];
    R.on_device = 1;
    R.n_contacts = bb_contacts + ss->contacts_f;
    const CellBox& nb = ss->next;
    bool inside = nb.bad == 0;
    for (int a = 0; a < 3; ++a) inside = inside && nb.lo[a] >= env.lo[a] && nb.hi[a] <= env.hi[a];
    if (ss->err) ctl->stop = GRAPH_STOP_ERROR;
    else if (!inside) ctl->stop = GRAPH_STOP_LEFT;
    ctl->step++;
    ctl->left--;
}

}  // namespace sphk
