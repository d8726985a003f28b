// sph_order.cuh — sorted order <-> caller order: the layout, and the only kernels that cross it.
// sph_kernels.cuh includes it next to sph_lists.cuh; the host side is export_rows / import_rows in sph_engine.cu.
//
// Every per-particle device array is in sorted cell order; the C ABI speaks caller order: the rows of the fluids (or of the
// boundaries) one after another, fluid f's rows starting at its offset.  orig[s] is the caller row of sorted slot s.
// A copy runs over a slot range [s0, s0 + n): the slots this GPU owns for fluids (s0 = own_begin, n = N; a slab world's
// ghosts lie outside it), every slot for boundaries (s0 = 0, n = B).  A column of `width` values per particle moves value k
// of slot s to dst[width * orig[s] + k] (export), or back from the packed rows [lo, hi) (import).
#pragma once

namespace sphk {

// Source views of an export: value k < width of sorted slot s, as the exported element type T.
struct Xyz {  // float4 x, y, z
    using T = float;
    static constexpr uint32_t width = 3;
    const float4* p;
    __device__ __forceinline__ float operator()(uint32_t s, uint32_t k) const {
        const float4 v = __ldg(p + s);  // one 16-byte load for the three values
        return k == 0 ? v.x : k == 1 ? v.y : v.z;
    }
};
struct W4 {  // float4 .w
    using T = float;
    static constexpr uint32_t width = 1;
    const float4* p;
    __device__ __forceinline__ float operator()(uint32_t s, uint32_t) const { return p[s].w; }
};
template <uint32_t W>
struct Rows {  // row-major, W floats per slot
    using T = float;
    static constexpr uint32_t width = W;
    const float* p;
    __device__ __forceinline__ float operator()(uint32_t s, uint32_t k) const { return p[(size_t)W * s + k]; }
};
struct Planes {  // `width` planes of `stride` floats
    using T = float;
    uint32_t width, stride;
    const float* p;
    __device__ __forceinline__ float operator()(uint32_t s, uint32_t k) const { return p[(size_t)k * stride + s]; }
};
template <class E>
struct U32 {  // a u32 column, exported as u32 (ids) or converted to E (contact counts)
    using T = E;
    static constexpr uint32_t width = 1;
    const uint32_t* p;
    __device__ __forceinline__ E operator()(uint32_t s, uint32_t) const { return (E)p[s]; }
};

// sorted slots [s0, s0 + n) -> caller rows of dst; a null orig maps slot s to row s
template <class V>
__global__ void k_export(uint32_t n, uint32_t s0, const uint32_t* __restrict__ orig, V src, typename V::T* __restrict__ dst) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t s = s0 + t;
    const size_t g = orig ? orig[s] : s;
#pragma unroll
    for (uint32_t k = 0; k < src.width; ++k) dst[src.width * g + k] = src(s, k);
}

// packed xyz rows [lo, hi) (row lo first) -> the sorted slots [s0, s0 + n) that hold them; slots of other rows are left
// alone.  Any source may be null: mass goes to pos.w and the fluid id's bits to vel.w only with their vector; vc gets w = 0.
__global__ void k_import(uint32_t n, uint32_t s0, const uint32_t* __restrict__ orig, const float* __restrict__ row_pos, const float* __restrict__ row_vel,
                         const float* __restrict__ row_vc, const float* __restrict__ row_mass, const uint32_t* __restrict__ row_fid, float4* __restrict__ pos,
                         float4* __restrict__ vel, float4* __restrict__ vc, uint32_t lo, uint32_t hi) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t s = s0 + t, g = orig[s];
    if (g < lo || g >= hi) return;
    const size_t r = g - lo;
    if (row_pos) {
        float4 p = pos[s];
        p.x = row_pos[3 * r]; p.y = row_pos[3 * r + 1]; p.z = row_pos[3 * r + 2];
        if (row_mass) p.w = row_mass[r];
        pos[s] = p;
    }
    if (row_vel) {
        float4 v = vel[s];
        v.x = row_vel[3 * r]; v.y = row_vel[3 * r + 1]; v.z = row_vel[3 * r + 2];
        if (row_fid) v.w = __uint_as_float(row_fid[r]);
        vel[s] = v;
    }
    if (row_vc) vc[s] = make_float4(row_vc[3 * r], row_vc[3 * r + 1], row_vc[3 * r + 2], 0.f);
}

}  // namespace sphk
