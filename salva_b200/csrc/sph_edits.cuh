// Particle sources and sinks (DESIGN.md section 14): the kernels that remove fluid particles inside sink boxes and append
// source templates at the start of a step, without restaging the world through the host.  faucet3.rs:69-105 does the same
// with delete_particle_at_next_timestep / add_particles from a host callback; fluid.rs:88-98, 126-150 give the order rules.
//
// One classification pass tests every slot against its fluid's sinks, writes keep flags (slot order) and removed flags
// (original order), and reduces per fluid the removals and 1 + the largest id, and the survivors' cell AABB as k_bounds
// computes it.  When anything is removed, both flag arrays are scanned together (scan_exclusive_k), k_edit_compact turns
// them into the gather's perm, the survivors' new original indices and the removed original indices, and k_gather moves
// the carried columns into the other parity.  A firing source is one k_edit_emit launch.
#pragma once
#include "sph_kernels.cuh"

namespace sphk {

constexpr int MAX_SINKS = 64, MAX_SOURCES = 64;  // per world (include/sph.h)

struct SinkBox {
    float lo[3], hi[3];
    int32_t outside;  // 1: removes what is NOT in the box
    uint32_t fluid;   // fluid slot
};
struct SinkSet {
    SinkBox b[MAX_SINKS];
    int n;
};
// what the classification reduces, read back with one copy
struct EditScan {
    unsigned long long next_id[MAX_FLUIDS];  // 1 + the largest id per fluid, 0 for an empty fluid
    uint32_t removed[MAX_FLUIDS];
    CellBox bounds;  // the survivors' cell box
};

// In the box iff lo <= x < hi on every axis: plain f32 comparisons, so NaN is in no box.
__device__ __forceinline__ bool sink_removes(const SinkBox& b, const float4& p) {
    const bool in = b.lo[0] <= p.x && p.x < b.hi[0] && b.lo[1] <= p.y && p.y < b.hi[1] && b.lo[2] <= p.z && p.z < b.hi[2];
    return b.outside ? !in : in;
}

// One thread per slot [0, n).  keep[s] (slot order) and removed[orig[s]] (original order) are 0 / 1.  Launch with 256 threads.
__global__ void k_edit_classify(uint32_t n, const float4* __restrict__ pos, const float4* __restrict__ vel, const uint32_t* __restrict__ gid,
                                const uint32_t* __restrict__ orig, const __grid_constant__ SinkSet sinks, uint32_t* __restrict__ keep,
                                uint32_t* __restrict__ removed, EditScan* __restrict__ out) {
    __shared__ unsigned long long s_next[MAX_FLUIDS];
    __shared__ uint32_t s_rm[MAX_FLUIDS];
    if (threadIdx.x < MAX_FLUIDS) {
        s_next[threadIdx.x] = 0ull;
        s_rm[threadIdx.x] = 0u;
    }
    __syncthreads();
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = s < n;
    bool rm = false;
    uint32_t f = 0u, g = 0u;
    CellBox b = CELL_BOX_EMPTY;
    if (valid) {
        const float4 p = pos[s];
        f = fid_of(vel[s]);
        g = gid[s];
        for (int k = 0; k < sinks.n && !rm; ++k) rm = sinks.b[k].fluid == f && sink_removes(sinks.b[k], p);
        keep[s] = rm ? 0u : 1u;
        removed[orig[s]] = rm ? 1u : 0u;
        if (!rm) cell_box_add(b, p.x, p.y, p.z, C.h);
    }
    // per fluid present in the warp: one shared atomic for its removals and one for its largest id
    const int lane = threadIdx.x & 31;
    for (unsigned pending = __ballot_sync(0xffffffffu, valid); pending;) {
        const int leader = __ffs((int)pending) - 1;
        const uint32_t lf = __shfl_sync(0xffffffffu, f, leader);
        const bool mine = valid && f == lf;
        const unsigned grp = __ballot_sync(0xffffffffu, mine);
        const uint32_t gmax = __reduce_max_sync(0xffffffffu, mine ? g : 0u);
        const uint32_t nrm = (uint32_t)__popc(__ballot_sync(0xffffffffu, mine && rm));
        if (lane == leader) {
            atomicMax(&s_next[lf], (unsigned long long)gmax + 1ull);
            if (nrm) atomicAdd(&s_rm[lf], nrm);
        }
        pending &= ~grp;
    }
    cell_box_commit_block(b, &out->bounds);  // (its barrier also ends the shared atomics above)
    if (threadIdx.x < MAX_FLUIDS) {
        if (s_next[threadIdx.x]) atomicMax(&out->next_id[threadIdx.x], s_next[threadIdx.x]);
        if (s_rm[threadIdx.x]) atomicAdd(&out->removed[threadIdx.x], s_rm[threadIdx.x]);
    }
}

// After the exclusive scans of keep (slot order) and removed (original order), both n + 1 long: a survivor in slot s goes to
// slot keep[s] (perm, for k_gather) and its original index o drops by the removals before it (fluid.rs:88-98 keeps the
// survivors' order); a removed particle writes o to its rank in the ascending list of removed original indices.
__global__ void k_edit_compact(uint32_t n, const uint32_t* __restrict__ keep, const uint32_t* __restrict__ removed, uint32_t* __restrict__ orig,
                               uint32_t* __restrict__ perm, uint32_t* __restrict__ removed_list) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t o = orig[s], k = keep[s];
    if (keep[s + 1] != k) {
        perm[k] = s;
        orig[s] = o - removed[o];
    } else {
        removed_list[removed[o]] = o;
    }
}

// A source's firing, as k_import would stage sph_fluid_append(template): slots [n, n + m) get the template with mass in
// pos.w, the fluid slot in vel.w, vc 0, ids id0.., IISPH pressure 0 and original indices end.. (the end of the fluid's
// range); the particles of the later fluids, original index >= end, move up by m.  max(n, m) threads.
__global__ void k_edit_emit(uint32_t n, uint32_t m, uint32_t end, const float4* __restrict__ tpos, const float4* __restrict__ tvel, float mass,
                            uint32_t fluid, uint32_t id0, float4* __restrict__ pos, float4* __restrict__ vel, float4* __restrict__ vc,
                            uint32_t* __restrict__ orig, uint32_t* __restrict__ gid, float* __restrict__ press) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) {
        const uint32_t o = orig[t];
        if (o >= end) orig[t] = o + m;
    }
    if (t < m) {
        const uint32_t s = n + t;
        const float4 p = tpos[t];
        const float4 v = tvel ? tvel[t] : make_float4(0.f, 0.f, 0.f, 0.f);
        pos[s] = make_float4(p.x, p.y, p.z, mass);
        vel[s] = make_float4(v.x, v.y, v.z, __uint_as_float(fluid));
        vc[s] = make_float4(0.f, 0.f, 0.f, 0.f);
        orig[s] = end + t;
        gid[s] = id0 + t;
        if (press) press[s] = 0.f;
    }
}

}  // namespace sphk
