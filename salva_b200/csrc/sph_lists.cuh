// sph_lists.cuh — the neighbour lists ("contacts", contacts.rs:83-87): their layout, and the only code that addresses them.
// sph_kernels.cuh includes it right after the constants: the addresses use C.stride, the counts C.cap_f / C.cap_b.
//
// The lists are index-only and column-major: column i belongs to particle slot i (sorted order), and a row holds
// C.stride entries (the world's per-particle plane stride, >= n_fluid, a multiple of 32).  The fluid list of particle i holds
// the sorted indices of its fluid neighbours, self included, ascending j, in one of two widths chosen per neighbour search
// (ListsOut::wide, DESIGN.md §4a.18):
//   wide (32-bit entries): nbr_f[((k / 4) * stride + i) * 4 + k % 4] = the k-th entry: groups of 4 contacts are interleaved so
//     a thread fetches 4 indices with one coalesced LDG.128; the tail slots of the last group hold i itself (a self contact
//     has zero gradient);
//   narrow (16-bit entries; the h-cell search of a one-GPU world): the candidates of a particle in cell (cx, cy, cz) that lie
//     in the x-plane cx + d - 1 (d = 0, 1, 2) are the cells (cx + d - 1, cy-1..cy+1, cz-1..cz+1), which in x-major, z-fastest
//     order lie in ONE slot range, the plane's window [cstart[cell(cx+d-1, cy-1, cz-1)], cstart[cell(cx+d-1, cy+1, cz-1) + 3]).
//       bases:   nbr_f[d * stride + i] = base_d, the first slot of window d;
//       entries: reinterpret_cast<uint2*>(nbr_f + 3 * stride)[(k / 4) * stride + i] holds entries 4 (k / 4) .. +3, 16 bits
//                each, low half first (one coalesced LDG.64 per group of 4): entry = d << 14 | (j - base_d), so
//                j = base[entry >> 14] + (entry & 0x3FFF).  The tail slots of the last group encode i in its own plane
//                (d = 1): every stored slot decodes to a contact or to i, and no count is needed to decode.
//     A search writes narrow lists only if every window of every particle spans at most WINDOW_SLOTS slots; otherwise it
//     raises StepScalars::max_nb[2] and the step repeats the search with wide lists.  Narrow lists take 3 + cap/2 words of
//     32 bits per particle and wide ones cap, so the same allocation holds either (cap_f >= 16).
//   nbr_b[k * stride + i] = the k-th boundary entry (32 bits, either width);
//   cnt_f[i], cnt_b[i] = the contacts the search found, which may exceed the capacities C.cap_f / C.cap_b (rows, multiples
//     of 16): only the first cap entries are stored, and a search past a capacity is run again with larger lists.
// W and grad W are recomputed from pos4 in every pass (cheaper than streaming cached 16-byte contacts from HBM: see DESIGN.md).
#pragma once

namespace sphk {

constexpr uint32_t WINDOW_SLOTS = 1u << 14;  // the most slots a narrow list's plane window may span (14-bit offsets)
// The generic-kernel library stores wide lists only: its gather passes have no registers to spare for the window bases.
#ifdef SPH_GENERIC_KERNELS
constexpr bool NARROW_LISTS = !SPH_GENERIC_KERNELS;
#else
constexpr bool NARROW_LISTS = true;
#endif

__device__ __forceinline__ size_t fluid_slot(uint32_t i, uint32_t k) { return ((size_t)(k >> 2) * C.stride + i) * 4 + (k & 3); }
__device__ __forceinline__ size_t boundary_slot(uint32_t i, uint32_t k) { return (size_t)k * C.stride + i; }
// how many of n found contacts a list stores
__device__ __forceinline__ uint32_t fluid_stored(uint32_t n) { return min(n, C.cap_f); }
__device__ __forceinline__ uint32_t boundary_stored(uint32_t n) { return min(n, C.cap_b); }

// A narrow list's three window bases
struct Window {
    uint32_t base[3];
    __device__ __forceinline__ uint32_t id(uint32_t e) const { return (e < 0x4000u ? base[0] : e < 0x8000u ? base[1] : base[2]) + (e & 0x3FFFu); }
    // the entry of j, a slot inside one of the windows
    __device__ __forceinline__ uint32_t entry(uint32_t j) const {
        const uint32_t d = j >= base[2] ? 2u : j >= base[1] ? 1u : 0u;
        return d << 14 | ((j - base[d]) & 0x3FFFu);
    }
    __device__ __forceinline__ uint4 ids(uint2 r) const { return make_uint4(id(r.x & 0xFFFFu), id(r.x >> 16), id(r.y & 0xFFFFu), id(r.y >> 16)); }
};
// narrow entries: uint2 groups past the three base rows
__device__ __forceinline__ size_t narrow_group(uint32_t i, uint32_t q) { return (size_t)q * C.stride + i; }

// One particle's fluid list as a gather pass walks it: raw(q) loads group q (4 entries, prefetched a group ahead as Raw),
// ids(raw) turns it into the 4 sorted indices.  n = the stored count; nq = (n + 3) / 4 groups.
struct WideRow {
    const uint4* p;  // group 0 of particle i
    uint32_t n;
    __device__ __forceinline__ uint4 raw(uint32_t q) const { return __ldcs(p + (size_t)q * C.stride); }
    __device__ __forceinline__ uint4 ids(uint4 r) const { return r; }
};
struct NarrowRow {
    const uint2* p;
    uint32_t n;
    Window w;
    __device__ __forceinline__ uint2 raw(uint32_t q) const { return __ldcs(p + (size_t)q * C.stride); }
    __device__ __forceinline__ uint4 ids(uint2 r) const { return w.ids(r); }
};

// The read view, passed to every gather pass.
struct Lists {
    const uint32_t* nbr_f;
    const uint32_t* nbr_b;
    const uint32_t* cnt_f;
    const uint32_t* cnt_b;
    bool wide;

    __device__ __forceinline__ uint32_t fluid_count(uint32_t i) const { return fluid_stored(cnt_f[i]); }
    __device__ __forceinline__ uint32_t boundary_count(uint32_t i) const { return boundary_stored(cnt_b[i]); }
    // every contact the search found, stored or not: what min_neighbors_for_divergence_solve compares (dfsph_solver.rs:301-314)
    __device__ __forceinline__ uint32_t gate_count(uint32_t i) const { return cnt_f[i] + cnt_b[i]; }
    __device__ __forceinline__ Window window(uint32_t i) const {
        return {{__ldcs(&nbr_f[i]), __ldcs(&nbr_f[C.stride + i]), __ldcs(&nbr_f[2 * (size_t)C.stride + i])}};
    }
    // f(row) with particle i's fluid list as a WideRow or a NarrowRow.  A pass streams its lists exactly once: they are loaded
    // with the evict-first policy so they do not push the gathered particle data out of L1/L2.
    template <class F>
    __device__ __forceinline__ void fluid_row(uint32_t i, F f) const {
        const uint32_t n = fluid_count(i);
        if (!NARROW_LISTS || wide) f(WideRow{reinterpret_cast<const uint4*>(nbr_f) + i, n});
        else f(NarrowRow{reinterpret_cast<const uint2*>(nbr_f + 3 * (size_t)C.stride) + i, n, window(i)});
    }
    // fluid entry k (below the count) on its own
    __device__ __forceinline__ uint32_t fluid(uint32_t i, uint32_t k) const {
        if (!NARROW_LISTS || wide) return nbr_f[fluid_slot(i, k)];
        const uint16_t e = reinterpret_cast<const uint16_t*>(nbr_f + 3 * (size_t)C.stride)[narrow_group(i, k >> 2) * 4 + (k & 3)];
        return window(i).id(e);
    }
    __device__ __forceinline__ uint32_t boundary(uint32_t i, uint32_t k) const { return nbr_b[boundary_slot(i, k)]; }
};

// The write view, passed to the neighbour search.  Entries past a capacity are dropped (the count still records them).
struct ListsOut {
    uint32_t* nbr_f;
    uint32_t* nbr_b;
    uint32_t* cnt_f;
    uint32_t* cnt_b;
    bool wide;

    // fluid entry k = j, in window d whose base is `base` (narrow)
    __device__ __forceinline__ void fluid(uint32_t i, uint32_t k, uint32_t j, uint32_t d, uint32_t base) const {
        if (k >= C.cap_f) return;
        if (!NARROW_LISTS || wide) nbr_f[fluid_slot(i, k)] = j;
        else reinterpret_cast<uint16_t*>(nbr_f + 3 * (size_t)C.stride)[narrow_group(i, k >> 2) * 4 + (k & 3)] = (uint16_t)(d << 14 | ((j - base) & 0x3FFFu));
    }
    __device__ __forceinline__ void boundary(uint32_t i, uint32_t k, uint32_t j) const {
        if (k < C.cap_b) nbr_b[boundary_slot(i, k)] = j;
    }
    // a whole group of four fluid entries 4q .. 4q+3 (q below cap_f / 4) of a list of n: J holds the sorted indices of those
    // below n; the slots past n point at i
    __device__ __forceinline__ void group(uint32_t i, uint32_t q, uint4 J, uint32_t n, const Window& w) const {
        const uint32_t k = q * 4u;
        J = make_uint4(J.x, k + 1 < n ? J.y : i, k + 2 < n ? J.z : i, k + 3 < n ? J.w : i);
        if (!NARROW_LISTS || wide) reinterpret_cast<uint4*>(nbr_f)[(size_t)q * C.stride + i] = J;
        else reinterpret_cast<uint2*>(nbr_f + 3 * (size_t)C.stride)[narrow_group(i, q)] = make_uint2(w.entry(J.x) | w.entry(J.y) << 16, w.entry(J.z) | w.entry(J.w) << 16);
    }
    // the tail of the last group of n fluid contacts, from entry `from` on, pointed at i
    __device__ __forceinline__ void pad(uint32_t i, uint32_t from, uint32_t n, const Window& w) const {
        for (uint32_t t = from; t < ((n + 3u) & ~3u) && t < C.cap_f; ++t) fluid(i, t, i, 1u, w.base[1]);
    }
    // the window bases of a narrow list
    __device__ __forceinline__ void bases(uint32_t i, const Window& w) const {
#pragma unroll
        for (int d = 0; d < 3; ++d) nbr_f[d * (size_t)C.stride + i] = w.base[d];
    }
    __device__ __forceinline__ void counts(uint32_t i, uint32_t nf, uint32_t nb) const {
        cnt_f[i] = nf;
        cnt_b[i] = nb;
    }
    __host__ __device__ Lists view() const { return {nbr_f, nbr_b, cnt_f, cnt_b, wide}; }
    // group q of particle i's fluid list as stored above, as sorted indices (this thread's own stores)
    __device__ __forceinline__ uint4 group_ids(uint32_t i, uint32_t q) const {
        if (!NARROW_LISTS || wide) return __ldcs(reinterpret_cast<const uint4*>(nbr_f) + (size_t)q * C.stride + i);
        return view().window(i).ids(__ldcs(reinterpret_cast<const uint2*>(nbr_f + 3 * (size_t)C.stride) + narrow_group(i, q)));
    }
};

}  // namespace sphk
