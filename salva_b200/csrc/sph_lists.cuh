// sph_lists.cuh — the neighbour lists ("contacts", contacts.rs:83-87): their layout, and the only code that addresses them.
// sph_kernels.cuh includes it right after the constants: the addresses use C.stride, the counts C.cap_f / C.cap_b.
//
// The lists are index-only and column-major: column i belongs to particle slot i (sorted order), and a row holds
// C.stride entries (the world's per-particle plane stride, >= n_fluid, a multiple of 32):
//   nbr_f[((k / 4) * stride + i) * 4 + k % 4] = sorted index of the k-th fluid neighbour of i (self included, ascending j):
//     groups of 4 contacts are interleaved so a thread fetches 4 indices with one coalesced LDG.128; the tail slots of the
//     last group hold i itself (a self contact has zero gradient);
//   nbr_b[k * stride + i] likewise (scalar) for boundary particles;
//   cnt_f[i], cnt_b[i] = the contacts the search found, which may exceed the capacities C.cap_f / C.cap_b (rows, multiples
//     of 16): only the first cap entries are stored, and a search past a capacity is run again with larger lists.
// W and grad W are recomputed from pos4 in every pass (cheaper than streaming cached 16-byte contacts from HBM: see DESIGN.md).
#pragma once

namespace sphk {

__device__ __forceinline__ size_t fluid_slot(uint32_t i, uint32_t k) { return ((size_t)(k >> 2) * C.stride + i) * 4 + (k & 3); }
__device__ __forceinline__ size_t boundary_slot(uint32_t i, uint32_t k) { return (size_t)k * C.stride + i; }
// how many of n found contacts a list stores
__device__ __forceinline__ uint32_t fluid_stored(uint32_t n) { return min(n, C.cap_f); }
__device__ __forceinline__ uint32_t boundary_stored(uint32_t n) { return min(n, C.cap_b); }

// The read view, passed to every gather pass.
struct Lists {
    const uint4* nbr_f;
    const uint32_t* nbr_b;
    const uint32_t* cnt_f;
    const uint32_t* cnt_b;

    __device__ __forceinline__ uint32_t fluid_count(uint32_t i) const { return fluid_stored(cnt_f[i]); }
    __device__ __forceinline__ uint32_t boundary_count(uint32_t i) const { return boundary_stored(cnt_b[i]); }
    // every contact the search found, stored or not: what min_neighbors_for_divergence_solve compares (dfsph_solver.rs:301-314)
    __device__ __forceinline__ uint32_t gate_count(uint32_t i) const { return cnt_f[i] + cnt_b[i]; }
    // fluid contacts 4q .. 4q+3.  A pass streams its lists exactly once: they are loaded with the evict-first policy so they
    // do not push the gathered particle data out of L1/L2.
    __device__ __forceinline__ uint4 group(uint32_t i, uint32_t q) const { return __ldcs(&nbr_f[(size_t)q * C.stride + i]); }
    __device__ __forceinline__ uint32_t fluid(uint32_t i, uint32_t k) const { return reinterpret_cast<const uint32_t*>(nbr_f)[fluid_slot(i, k)]; }
    __device__ __forceinline__ uint32_t boundary(uint32_t i, uint32_t k) const { return nbr_b[boundary_slot(i, k)]; }
};

// The write view, passed to the neighbour search.  Entries past a capacity are dropped (the count still records them).
struct ListsOut {
    uint32_t* nbr_f;
    uint32_t* nbr_b;
    uint32_t* cnt_f;
    uint32_t* cnt_b;

    __device__ __forceinline__ void fluid(uint32_t i, uint32_t k, uint32_t j) const {
        if (k < C.cap_f) nbr_f[fluid_slot(i, k)] = j;
    }
    __device__ __forceinline__ void boundary(uint32_t i, uint32_t k, uint32_t j) const {
        if (k < C.cap_b) nbr_b[boundary_slot(i, k)] = j;
    }
    // a whole group of four fluid entries, 4q .. 4q+3 (q below cap_f / 4)
    __device__ __forceinline__ void group(uint32_t i, uint32_t q, uint4 J) const { reinterpret_cast<uint4*>(nbr_f)[(size_t)q * C.stride + i] = J; }
    // the tail of the last group of n fluid contacts, from entry `from` on, pointed at i itself
    __device__ __forceinline__ void pad(uint32_t i, uint32_t from, uint32_t n) const {
        for (uint32_t t = from; t < ((n + 3u) & ~3u) && t < C.cap_f; ++t) nbr_f[fluid_slot(i, t)] = i;
    }
    __device__ __forceinline__ void counts(uint32_t i, uint32_t nf, uint32_t nb) const {
        cnt_f[i] = nf;
        cnt_b[i] = nb;
    }
    __host__ __device__ Lists view() const { return {reinterpret_cast<const uint4*>(nbr_f), nbr_b, cnt_f, cnt_b}; }
};

}  // namespace sphk
