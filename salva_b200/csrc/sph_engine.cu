// sph_engine.cu — world state, step driver and the extern "C" boundary (include/sph.h) of the
// H100-native SPH step path.  The step sequence restates LiquidWorld::step_with_coupling
// (liquid_world.rs:67-158) + DFSPHSolver::step (dfsph_solver.rs:667-708) / IISPHSolver::step
// (iisph_solver.rs:643-711) as a chain of CUDA kernels on one stream; see DESIGN.md.
//
// There is no CPU fallback: every entry point needs a CUDA device.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/sph.h"
#include "sph_kernels.cuh"
#include "sph_shapes.cuh"
#include "sph_passes.cuh"
#include "sph_iisph.cuh"
#include "sph_elasticity.cuh"
#include "sph_viscosity.cuh"
#include "sph_sampling.cuh"
#include "sph_edits.cuh"
#include "sph_surface.cuh"
#include "sph_diffuse.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

using namespace sphk;

namespace {

// All worlds of a process share the module's __constant__ block; API calls are serialised per process
// (GPU work of different worlds on one device would serialise anyway) and re-upload it on entry.
// recursive: host-force and coupling callbacks run inside sph_world_step and may call back into the API (reads,
// boundary rewrites, queries) on the same thread
std::recursive_mutex g_mutex;
const void* g_const_owner = nullptr;

inline uint32_t cdiv(size_t a, size_t b) { return (uint32_t)((a + b - 1) / b); }

// A device buffer that owns its allocation: it moves, never copies, and frees the allocation when it dies.
template <class T>
struct DBuf {
    T* p = nullptr;
    size_t cap = 0;
    DBuf() = default;
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    DBuf(DBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DBuf& operator=(DBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = std::exchange(o.p, nullptr);
            cap = std::exchange(o.cap, 0);
        }
        return *this;
    }
    ~DBuf() { release(); }
    cudaError_t ensure(size_t n, bool keep = false, cudaStream_t st = 0) {
        if (n <= cap) return cudaSuccess;
        size_t ncap = std::max(n, cap + cap / 4);
        T* q = nullptr;
        cudaError_t e = cudaMalloc(&q, ncap * sizeof(T));
        if (e != cudaSuccess) return e;
        if (keep && p && cap) {
            e = cudaMemcpyAsync(q, p, cap * sizeof(T), cudaMemcpyDeviceToDevice, st);
            if (e != cudaSuccess) return e;
            cudaStreamSynchronize(st);
        }
        if (p) cudaFree(p);
        p = q;
        cap = ncap;
        return cudaSuccess;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

// A linear texture object over a DBuf, destroyed with its owner; declare it after the buffer it views.
struct Tex {
    cudaTextureObject_t obj = 0;
    const void* ptr = nullptr;
    size_t bytes = 0;
    Tex() = default;
    Tex(const Tex&) = delete;
    Tex& operator=(const Tex&) = delete;
    ~Tex() {
        if (obj) cudaDestroyTextureObject(obj);
    }
    // rebuilds the object only when the buffer's allocation changed
    template <class T>
    cudaError_t bind(const DBuf<T>& b) {
        if (obj && ptr == b.p && bytes == b.cap * sizeof(T)) return cudaSuccess;
        if (obj) cudaDestroyTextureObject(obj);
        obj = 0;
        cudaResourceDesc rd;
        memset(&rd, 0, sizeof rd);
        rd.resType = cudaResourceTypeLinear;
        rd.res.linear.devPtr = b.p;
        rd.res.linear.desc = cudaCreateChannelDesc<T>();
        rd.res.linear.sizeInBytes = b.cap * sizeof(T);
        cudaTextureDesc td;
        memset(&td, 0, sizeof td);
        td.readMode = cudaReadModeElementType;
        cudaError_t e = cudaCreateTextureObject(&obj, &rd, &td, nullptr);
        if (e != cudaSuccess) {
            obj = 0;
            return e;
        }
        ptr = b.p;
        bytes = b.cap * sizeof(T);
        return cudaSuccess;
    }
};

// The neighbour lists (layout: sph_lists.cuh) and their capacities in rows.  The constants carry the capacities: grow_lists()
// raises them.
struct ListState {
    DBuf<uint32_t> nbr_f, nbr_b, cnt_f, cnt_b;
    uint32_t cap_f = 64, cap_b = 32;
    Lists view() const { return out().view(); }
    ListsOut out() const { return {nbr_f.p, nbr_b.p, cnt_f.p, cnt_b.p}; }
    // counts for n particles, and cap_f / cap_b rows of `stride` entries (sph_world::stride)
    cudaError_t ensure(size_t n, uint32_t stride) {
        cudaError_t e = cnt_f.ensure(n);
        if (e == cudaSuccess) e = cnt_b.ensure(n);
        if (e == cudaSuccess) e = nbr_f.ensure((size_t)cap_f * stride);
        if (e == cudaSuccess) e = nbr_b.ensure((size_t)cap_b * stride);
        return e;
    }
};

// Solver and plugin scratch.  The kernels take the raw pointers (.p).
struct IisphState {
    DBuf<float4> dii;      // iisph_solver.rs:32
    DBuf<float4> dij_pjl;  // iisph_solver.rs:34
    DBuf<float4> s;        // dii * p + dij_pjl
    DBuf<float> aii;       // iisph_solver.rs:33
    DBuf<float> next_p;    // iisph_solver.rs:38
    DBuf<float> prho;      // p / rho^2
    DBuf<float> next_prho;
    size_t cap = 0;        // rows of every buffer; 0 until all of them are allocated
    Tex tex_s;             // over s
};
struct ViscosityState {
    DBuf<float> beta;    // beta[(r * 6 + c) * stride + i]
    DBuf<float> target;  // target[k * stride + i]            dfsph_viscosity.rs:24
    DBuf<float4> vv;     // vel + acc * dt
    DBuf<float4> u4;     // u[0..3]
    DBuf<float2> u2;     // u[4..5]
    size_t cap = 0;      // rows of every buffer; 0 until all of them are allocated
};
// Becker2009 rest pose of one force (sph_elasticity_host.inl)
struct ElasticityState {
    size_t n = 0;            // particle count the rest pose was captured for (re-captured when it changes, :87)
    uint32_t cap0 = 0;       // rest-list capacity (rows)
    uint32_t stride0 = 0;
    DBuf<float4> pos0;       // positions0.xyz, volumes0 in .w
    DBuf<uint32_t> nbr0;     // nbr0[k * stride0 + t]: local original index of the k-th rest contact (self included)
    DBuf<uint32_t> cnt0;
    DBuf<float> rot;         // 9 floats per particle, row-major rotation (warm start for the next step, :134-135)
    DBuf<float> grad_tr;     // 9 floats per particle: deformation_gradient_tr
    DBuf<float> stress;      // 6 floats per particle: x y z w a b (:27-37)
    DBuf<float4> cur;        // current positions (xyz) + mass (.w) in original order
    DBuf<uint32_t> slot_of;  // sorted slot of local original index t
    float d0 = 0.f, d1 = 0.f, d2 = 0.f;
};

// Fluid surface extraction (sph_surface_host.inl): the collected particles, their cells and the lattice scratch of one
// extraction, and the field and mesh of the last one.  An extraction builds into the scratch set and swaps it in on success,
// so a refused one keeps the previous mesh.
struct SurfaceSet {
    DBuf<float> phi, verts, nrm;
    DBuf<uint32_t> tris;
    SurfLattice L{};
    size_t nv = 0, nt = 0;
    bool normals = false;
    // an anisotropic extraction's ellipsoids (section 17), collected order: centre xyz, and (e1, a1, e2, a2, e3, a3)
    bool aniso = false;
    DBuf<float> ecen, eaxes;
    SurfSel esel{};
    uint32_t ehandle[MAX_FLUIDS] = {};  // the selected fluids' handles at the extraction (~0: not selected)
    uint32_t en[MAX_FLUIDS] = {};       // ... and their particle counts
};
struct SurfaceState {
    DBuf<uint32_t> vcnt, tcnt, scan_aux[3];
    DBuf<uint8_t> emask;
    DBuf<unsigned long long> totals;
    DBuf<float4> e4[3], se4[3];  // anisotropic: (x_bar, V h^3 / (a1 a2 a3)) and h G's six entries, collected, then in cell order
    SurfaceSet cur, next;
};
// The selected fluids' particles binned into cells of width h for one surface extraction or diffuse update
// (sph_surface_host.inl bins_collect / bins_sort).  Collected rows follow the fluids' index order, slot by slot (sel.out_off).
struct FluidBins {
    DBuf<float4> p4, sp4;          // (x, y, z, volume): collected, then in cell order
    DBuf<float4> v4, sv4;          // velocities (x, y, z, 0), when asked for: collected, then in cell order
    DBuf<unsigned long long> key;  // (fluid slot, id), collected order
    DBuf<float> vol;               // the host's volume column while it is not all default
    DBuf<uint32_t> cid, rank, perm, cstart, aabb, scan_aux[3];
    SurfSel sel{};
    SurfGrid g{};
    size_t np = 0, ncell = 0, binned = 0;  // collected, cells, binned (finite positions inside the cells)
    bool have = false;                     // some collected position is finite; then amin / amax is their AABB
    float amin[3] = {0.f, 0.f, 0.f}, amax[3] = {0.f, 0.f, 0.f};
};
// Diffuse particles (sph_diffuse_host.inl, DESIGN.md section 16).  A set in the published layout, with the per-fluid-particle
// values of the update that made it (collected order, for sph_debug_read); an update builds into `next` and swaps it in on
// success, so a refused one keeps the last set.
struct DiffuseSet {
    DBuf<float> pos, vel, life;  // packed xyz, xyz, life
    DBuf<uint8_t> kind;
    size_t n = 0;
    DBuf<float> nrm, ta, wc, ek;  // per collected fluid particle: normal (xyz), I_ta, I_wc, E_k
    DBuf<uint32_t> nd;            // ... and its emission count
    SurfSel sel{};                // the fluids those rows belong to
    uint32_t sel_n[MAX_FLUIDS] = {};
};
struct DiffuseState {
    DBuf<float4> nrm4;                 // normals of the binned fluid, cell order
    DBuf<unsigned long long> cnt, off;  // emission counts in cell order and their exclusive scan
    DBuf<char> scan_tmp;               // the offsets scan's scratch
    DBuf<float4> wx, wv;               // the advected set before compaction: (x, life), (v, kind bits)
    DBuf<uint32_t> keep, scan_aux[3];  // keep flags, scanned in place into output rows
    DBuf<unsigned long long> totals;   // expired, left the box, spray, foam, bubble
    uint32_t counter = 0;              // successful updates: the hash's update counter
    DiffuseSet cur, next;
};

struct ForceRec;
}  // namespace
struct sph_world;
namespace {
constexpr int FORCE_HOST_CALLBACK = 100;  // internal kind of sph_fluid_push_host_force entries
struct ForceRec {
    sph_force_desc d;
    sph_host_force_fn host_fn = nullptr;
    sph_host_force_fn2 host_fn2 = nullptr;  // context-style callback (contacts / boundaries on request)
    uint32_t host_flags = 0;
    void* host_user = nullptr;
    std::unique_ptr<ElasticityState> elastic;  // Becker2009 rest-pose state
    uint32_t visc_iters = 0;             // DFSPHViscosity: acceleration updates of the last solve
    float visc_err = 0.f;                // ... and its last strain-rate error
    bool solved = false;                 // has run in a step (sph_debug_read's plugin scratch is valid until particles change)
};
struct FluidRec {
    size_t n = 0, offset = 0;
    float density0 = 1000.f;
    uint32_t memberships = 1, filter = 0xFFFFFFFFu;
    std::vector<ForceRec> forces;
    std::vector<uint8_t> pending_delete;
    size_t n_pending = 0;
    float uniform_mass = 0.f;  // common particle mass if all volumes are equal, else 0
    bool alive = true;         // false after LiquidWorld::remove_fluid (liquid_world.rs:171-173); the slot is reused by the next add
    uint32_t gen = 0;          // handle = slot | gen << 16 (the reference's arena handles carry a generation too)
    size_t step_removed = 0, step_emitted = 0;  // what the last step's sinks removed and its sources emitted
    // move-only: the forces own device memory, and std::vector<ForceRec> would still declare a copy
    FluidRec() = default;
    FluidRec(FluidRec&&) = default;
    FluidRec& operator=(FluidRec&&) = default;
};
struct BoundaryRec {
    size_t n = 0, offset = 0;
    uint32_t memberships = 1, filter = 0xFFFFFFFFu;
    bool want_forces = false;
    bool alive = true;
    uint32_t gen = 0;
};

// fluid.rs:110-120: the volume of a particle given none
inline float default_volume(float r) { return r * r * r * (float)(8.0 * 0.8); }

// Rows [at, at + old) of a column with `width` values per row become n rows copied from src, or n rows of `fill`.
template <class T>
void splice_rows(std::vector<T>& c, size_t width, size_t at, size_t old, size_t n, const T* src, T fill) {
    c.erase(c.begin() + width * at, c.begin() + width * (at + old));
    if (src) c.insert(c.begin() + width * at, src, src + width * n);
    else c.insert(c.begin() + width * at, width * n, fill);
}

// Keeps the rows of a column whose mask entry is set, in order.
template <class T>
void keep_rows(std::vector<T>& c, size_t width, const std::vector<uint8_t>& mask) {
    size_t kept = 0;
    for (size_t i = 0; i < mask.size(); ++i)
        if (mask[i]) std::copy_n(c.begin() + width * i, width, c.begin() + width * kept++);
    c.resize(width * kept);
}

// What the fluid particles carry across steps, on the host in slot order (the fluids' ranges one after the other): the
// truth while sph_world::staged.  Every column holds one row per particle; host edits change rows through splice and keep.
struct FluidRows {
    std::vector<float> pos, vel, vc;  // xyz per row
    std::vector<float> vol, press;    // volume, IISPH pressure
    std::vector<uint32_t> gid;        // caller-visible id
    float vol0 = 0.f;                 // default_volume of the world's particle radius

    // Rows [at, at + old) become n new ones.  A null vel, vc or volume reads as zero, zero and vol0; pressures start at 0.
    void splice(size_t at, size_t old, size_t n, const float* p, const float* v, const float* c, const float* volume, const uint32_t* ids) {
        splice_rows(pos, 3, at, old, n, p, 0.f);
        splice_rows(vel, 3, at, old, n, v, 0.f);
        splice_rows(vc, 3, at, old, n, c, 0.f);
        splice_rows(vol, 1, at, old, n, volume, vol0);
        splice_rows(press, 1, at, old, n, (const float*)nullptr, 0.f);
        splice_rows(gid, 1, at, old, n, ids, 0u);
    }
    void keep(const std::vector<uint8_t>& mask) {
        keep_rows(pos, 3, mask);
        keep_rows(vel, 3, mask);
        keep_rows(vc, 3, mask);
        keep_rows(vol, 1, mask);
        keep_rows(press, 1, mask);
        keep_rows(gid, 1, mask);
    }
    // n rows for a download that writes positions, velocities, vc and ids.  Pressures read 0 until it writes them too;
    // volumes stay with their rows, and rows past the old size (a slab step's immigrants) take vol0.
    void resize(size_t n) {
        pos.resize(3 * n);
        vel.resize(3 * n);
        vc.resize(3 * n);
        vol.resize(n, vol0);
        press.assign(n, 0.f);
        gid.resize(n);
    }
    struct Column { void* p; size_t row_bytes; };
    // the columns in the order of a snapshot (format version 1)
    std::array<Column, 6> columns() {
        return {{{pos.data(), 3 * sizeof(float)}, {vel.data(), 3 * sizeof(float)}, {vc.data(), 3 * sizeof(float)},
                 {vol.data(), sizeof(float)}, {press.data(), sizeof(float)}, {gid.data(), sizeof(uint32_t)}}};
    }
};

// The boundary particles on the host in slot order; every column has as many rows as the boundaries have particles.
struct BoundaryRows {
    std::vector<float> pos, vel;  // xyz per row
    // rows [at, at + old) become n new ones; a null vel reads as zero
    void splice(size_t at, size_t old, size_t n, const float* p, const float* v) {
        splice_rows(pos, 3, at, old, n, p, 0.f);
        splice_rows(vel, 3, at, old, n, v, 0.f);
    }
    void resize(size_t n) {
        pos.resize(3 * n);
        vel.resize(3 * n);
    }
};
// ColliderCouplingEntry (fluids_pipeline.rs:76-80)
struct ColliderRec {
    uint32_t boundary = 0;          // boundary handle; a removed boundary leaves the collider inert
    int32_t sampling = SPH_SAMPLING_STATIC;
    sph_shape shape{};              // SPH_SAMPLING_CONTACT: the collider's shape
    size_t n = 0;                   // StaticSampling: sample points
    DBuf<float4> local;             // the points in the collider's frame
    DBuf<float> hgt;                // a heightfield shape (shape.kind == SPH_SHAPE_HEIGHTFIELD): its heights, owned by the record
    HfGrid hf{};                    // ... its grid constants (hf.hgt = hgt.p)
    float hf_ylo = 0.f, hf_yhi = 0.f;  // ... and its scaled height range: the local AABB's y extent
    sph_collider_state state{};     // for the next step
    sph_collider_state applied{};   // what the boundary's particles on the device were posed with
    bool applied_valid = false;
    float impulse[6] = {};          // of the last step: linear, angular
    bool impulse_pending = false;   // this step's reduction is in flight to sph_world::h_imp
    bool alive = true;
    uint32_t gen = 0;
};
// A particle sink or source of one fluid (sph_edits_host.inl); handles are slot | gen << 16 like the colliders'.
struct SinkRec {
    sph_sink_desc d{};
    uint32_t fluid = 0;  // fluid slot
    bool alive = true;
    uint32_t gen = 0;
};
struct SourceRec {
    uint32_t fluid = 0;
    size_t n = 0;             // template particles
    DBuf<float4> pos, vel;    // the template, uploaded at registration
    bool has_vel = false;
    uint32_t interval = 1, age = 0;  // fires on the steps with age % interval == 0; age counts the steps since registration
    CellBox cells = CELL_BOX_EMPTY;  // the template's cell box
    bool alive = true;
    uint32_t gen = 0;
};
static_assert(!std::is_copy_constructible<DBuf<float>>::value && !std::is_copy_constructible<ForceRec>::value &&
                  !std::is_copy_constructible<FluidRec>::value && !std::is_copy_constructible<ColliderRec>::value,
              "records that own device memory move, never copy");

sph_status iisph_step(sph_world* w, float dt_total, const float g[3]);
sph_status slab_begin_step(sph_world* w);
sph_status slab_after_sort(sph_world* w);
sph_status slab_refresh(sph_world* w, void* array, size_t elem);
struct SlabArray {
    void* p;
    size_t elem;
};
sph_status slab_refresh_n(sph_world* w, const SlabArray* arrays, int n_arrays);
sph_status p2p_setup(sph_world* w);
sph_status post_density_refresh(sph_world* w);
sph_status slab_allreduce(sph_world* w, float* buf, size_t n);
void slab_release(sph_world* w);
const float* iisph_pred(sph_world* w);
sph_status elasticity_solve(sph_world* w, uint32_t fluid, ForceRec& fr);
sph_status elasticity_restore(sph_world* w, ForceRec& fr, size_t n, uint32_t cap0, uint32_t stride0, const char* blob);
sph_status viscosity_solve(sph_world* w, uint32_t fluid, ForceRec& fr);
bool any_collider(const sph_world* w);
bool any_contact(const sph_world* w);
sph_status colliders_update(sph_world* w, bool reposed_all);
sph_status colliders_contact(sph_world* w);
sph_status colliders_impulse(sph_world* w);
bool any_edit(const sph_world* w);
sph_status edits_before_marks(sph_world* w, uint64_t* next);
sph_status apply_sources_sinks(sph_world* w, uint64_t* next);
inline float __uint_as_float_host(uint32_t u) {
    float f;
    memcpy(&f, &u, sizeof f);
    return f;
}

struct P2PState {  // NVLink peer-memory exchange (sph_slab.inl)
    bool on = false;
    size_t box_bytes = 0;
    char* base = nullptr;          // my landing zones + flags + reduction table (one cudaIpc-exported allocation)
    char* peer_base[8] = {};       // the same allocation of every rank, mapped into this process ([rank] == base)
    uint32_t seq_send[2] = {0, 0}, seq_recv[2] = {0, 0}, red_seq = 0;
    DBuf<uint32_t> tickets;
};

struct SlabState {
    bool active = false, own_comm = false;
    P2PState p2p;
    int rank = 0, nranks = 1;
    int lo = INT_MIN, hi = INT_MAX;  // owned cell columns [lo, hi) in absolute cell coordinates floor(x / h)
    int has_left = 0, has_right = 0;
    void* comm = nullptr;
    DBuf<uint32_t> d_cnt, flag, gid_l, gid_r, gid_cl, gid_cr;
    uint32_t cap_out = 1u << 14, cap_col = 1u << 17;  // staging capacities (emigrants / boundary-column particles per side); grown on demand
    uint32_t sort_off = 0, sort_n = 0, sort_dead_n = 0;  // what the step's counting sort reads (set by slab_begin_step)
    DBuf<unsigned long long> d_cnt64;
    DBuf<float4> out_l[3], out_r[3], col_l[3], col_r[3];
    bool global_valid = false;
    // slot ranges of the current step (after the sort)
    uint32_t gl_count = 0, sl_begin = 0, sl_count = 0, sr_begin = 0, sr_count = 0, gr_begin = 0, gr_count = 0;
    uint32_t exp_ghost_l = 0, exp_ghost_r = 0, exp_send_l = 0, exp_send_r = 0;
    uint32_t migrated_in = 0, migrated_out = 0;
    unsigned long long global_n = 0;
};

// sph_world_step_many's captured steps (sph_graph.inl): instantiated graphs, each with the state it was captured from
struct StepGraph {
    std::vector<char> key;
    cudaGraph_t g = nullptr;
    cudaGraphExec_t x = nullptr;
};
struct StepGraphs {
    std::vector<StepGraph> cache;       // at most one per parity of the fluid and the boundary buffers
    std::vector<cudaStream_t> streams;  // conditional bodies are captured on these, one per nesting level
    int depth = 0;
    DBuf<GraphCtl> ctl;
    DBuf<StepRec> rec;
    GraphCtl* h_ctl = nullptr;          // pinned
    cudaGraphConditionalHandle h_lists = 0;  // the IF of the step being captured past its neighbour search
    cudaGraph_t top = nullptr;          // the graph being captured
    CellBox env{};                      // the fluid cell range the graph's grid covers with ENVELOPE_MARGIN to spare
    bool env_valid = false;             // env was set up by an earlier call
    bool driver_checked = false;
    bool unsupported = false;           // the driver predates CUDA 12.4: step_many runs the per-step path
    void drop() {
        for (auto& e : cache) {
            if (e.x) cudaGraphExecDestroy(e.x);
            if (e.g) cudaGraphDestroy(e.g);
        }
        cache.clear();
    }
    void release() {
        drop();
        for (auto s : streams) cudaStreamDestroy(s);
        streams.clear();
        if (h_ctl) cudaFreeHost(h_ctl);
        h_ctl = nullptr;
    }
};

enum { EV_START = 0, EV_GRID, EV_NBR, EV_DENS, EV_DIV, EV_FOLD, EV_FORCES, EV_INTEG, EV_PRESS, EV_END, EV_COUNT };

}  // namespace

struct sph_world {
    sph_world_desc desc;
    float h = 0.f;
    cudaStream_t st = nullptr;
    cudaEvent_t ev[EV_COUNT] = {};
    cudaEvent_t ev_lists = nullptr;  // list-capacity read-back of phase_neighbors
    std::string err;
    Consts hc;

    std::vector<FluidRec> fluids;
    std::vector<BoundaryRec> bounds;
    size_t N = 0, B = 0;   // N = fluid particles OWNED by this world
    size_t Ntot = 0;       // slots of the sorted arrays during a step: owned + ghost (== N on one GPU)
    int protect_buf = -1;    // double-buffer index ensure_fluid_buffers() must not reallocate (it is being read)
    uint32_t own_begin = 0;  // first owned slot (ghost columns of a slab world sit at both ends of the sorted arrays)
    SlabState slab;
    uint64_t stats_exchanges = 0;

    // timestep_manager.rs:21-31: dt/inv_dt are 0 until the first advance()
    float dt = 0.f, inv_dt = 0.f;
    int force_div = -1, force_press = -1;
    // CFL-bounded substeps (sph_world_set_substepping, DESIGN.md section 12): off while cfl_coeff == 0
    float cfl_coeff = 0.f;
    uint32_t min_substeps = 1, max_substeps = 10;
    std::vector<float> substeps;  // dt_k of the last step's substeps, in order (its size is the running substep's k)

    // host truth in ORIGINAL order while `staged` (before the first step / after structural edits)
    bool staged = true;
    FluidRows rows;
    // boundaries: host copy is always kept (static data); b_dirty => re-upload
    bool b_dirty = true;
    CellBox b_box = CELL_BOX_EMPTY;  // the boundaries' cell box (host side, static)
    // the boundary sort / volumes are reused while the boundaries and the grid mapping are unchanged
    bool b_sorted_valid = false, b_reused = false;
    unsigned long long bb_contacts = 0;
    int b_sorted_grid[6] = {0, 0, 0, 0, 0, 0};
    BoundaryRows brows;
    bool hb_stale = false;  // colliders posed boundary particles on the device: brows lags behind (pull_boundaries)
    std::vector<ColliderRec> colliders;
    DBuf<CellBox> d_cb;     // the boundaries' cell box after colliders moved
    DBuf<float> d_imp;      // 6 floats per collider slot: the impulses of the step
    float* h_imp = nullptr;  // pinned copy, read back with the step's final read-back
    // DynamicContactSampling (colliders_contact): collider table, result ints, growing sample / push records, sort buffers
    DBuf<ContactCollider> d_ccol;
    DBuf<HfGrid> d_chf;  // per contact collider: a heightfield's grid (ContactParams::hf)
    DBuf<ContactResults> d_cres;
    DBuf<float4> cs_s4, cs_p4;
    DBuf<unsigned long long> cs_key[2];
    DBuf<uint32_t> cs_val[2];
    DBuf<char> cs_tmp;
    uint32_t cap_s = 4096, cap_p = 4096;
    // sph_world_sample_shape: ray tables + heights, per-ray counts / offsets, candidate keys, points, flags
    DBuf<float> smp_f, smp_xyz;
    DBuf<unsigned long long> smp_cnt, smp_off, smp_key[2];
    DBuf<int> smp_flag;

    // sorted device state (double buffered for the counting sort)
    int cur = 0, bcur = 0;
    DBuf<float4> pos[2], vel[2], vc[2], bpos[2], bvel[2];
    DBuf<uint32_t> orig[2], borig[2];
    DBuf<uint32_t> gid[2];  // caller-visible particle ids (default: original index); follow particles across ranks
    DBuf<float> press[2];
    DBuf<float4> vs, acc, normals, dbg_acc;
    DBuf<float> dens, alpha, kappa, divv, pred, bvol, bforce;
    DBuf<uint32_t> cid, rank, perm, cstart, bcid, brank, bperm, bstart, scan_aux[3], scan_aux_k[3];
    DBuf<unsigned long long> skey;  // deterministic mode: the in-cell sort keys beside perm / bperm (k_cell_scatter)
    ListState lists;
    // uniform-mass packed gather records (sph_passes.cuh): pvx4 = (x,y,z,v*x), vyz2 = (v*y,v*z), pk4 = (x,y,z,kappa); their
    // gathers are split evenly over the texture and LSU pipes (even / odd contacts)
    bool unimass = false;
    DBuf<float4> pvx4, pk4;
    DBuf<float2> vyz2;
    Tex tex_pvx, tex_vyz, tex_pk;
    DBuf<float> he_colors, he_gradc;  // He2014 colours / squared colour-gradient norms (he2014_surface_tension.rs:16-17)
    DBuf<uint32_t> q_out, q_count;     // particles_intersecting_aabb results
    DBuf<float> map_pos, map_vel;      // sph_fluid_map_positions / _velocities: ORIGINAL-order device views
    bool in_coupling = false;          // inside CouplingManager::update_boundaries: the grid holds fluids only (liquid_world.rs:90-103)
    bool in_host_force = false;        // inside a host NonPressureForce callback
    const sph_coupling_manager* coupling = nullptr;
    // ParticlesContacts materialised for host plugins (original order CSR)
    DBuf<uint32_t> ct_cnt[2], ct_j[2], ct_model[2];
    DBuf<float> ct_w[2], ct_g[2];
    DBuf<float4> xs;  // the XSPH sums or the Akinci fluid force of a divergence evaluation (fold_state)
    uint32_t fused_nblk = 0;
    Tex tex_vs;  // the general evaluations gather v* through the texture pipe
    DBuf<float> partial;
    DBuf<StepScalars> d_ss;
    StepScalars* h_ss = nullptr;  // pinned mirror of d_ss: every read-back lands in its own fields
    DBuf<uint32_t> rows_scratch;  // caller-order rows of export_rows / import_rows, one region per column
    IisphState iisph;
    ViscosityState visc;

    // fine-grained kernel timers: (slot, begin, end) event pairs accumulated into stats at step end
    struct Span { int slot; cudaEvent_t a, b; };
    std::vector<Span> spans;
    size_t n_spans = 0;

    uint32_t stride = 0;  // per-particle plane stride (Consts::stride)
    bool lists_valid = false;
    // cell-coordinate AABB of the positions the last step wrote (k_update_positions): sizes the next grid without a bounds pass
    bool nb_valid = false, nb_pending = false;
    CellBox nb = CELL_BOX_EMPTY;
    // particle sinks and sources (sph_edits_host.inl) and their classification's flags, result and removed original indices
    std::vector<SinkRec> sinks;
    std::vector<SourceRec> sources;
    DBuf<EditScan> d_edit;
    EditScan* h_edit = nullptr;  // pinned
    DBuf<uint32_t> ed_keep, ed_rm, ed_list;
    SurfaceState surf;  // sph_world_extract_surface's scratch and its last mesh
    FluidBins bins;     // the fluid binned for the last surface extraction or diffuse update
    DiffuseState diffuse;  // sph_world_update_diffuse's scratch and its set
    bool vol_all_default = true;  // every row of rows.vol is rows.vol0 (set by stage_up): edits then only resize the column
    int xysub = 1;              // row order (Consts::xysub, SALVA_B200_XYSUB): x / y bins per cell; one GPU only

    bool grid_ready = false;    // cstart/bstart + sorted arrays describe the last step's cell grid (AABB queries)
    bool ever_stepped = false;
    sph_step_stats stats;
    uint64_t launches = 0;
    uint32_t max_nb_b = 0;                 // the widest boundary list of the last neighbour search
    std::vector<sph_step_record> records;  // one per step of the last sph_world_step / sph_world_step_many call
    StepGraphs graphs;                     // sph_world_step_many's captured steps (sph_graph.inl)
    bool cap = false;                      // the launches go into a step graph: no host read-back, sync or event

    // Every DBuf, Tex and record frees itself after this body; it destroys what is not device memory.
    ~sph_world() {
        for (auto& s : spans) {
            cudaEventDestroy(s.a);
            cudaEventDestroy(s.b);
        }
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (ev_lists) cudaEventDestroy(ev_lists);
        graphs.release();
        if (h_ss) cudaFreeHost(h_ss);
        if (h_imp) cudaFreeHost(h_imp);
        if (h_edit) cudaFreeHost(h_edit);
        if (st) cudaStreamDestroy(st);
    }

    sph_status fail(sph_status s, const char* fmt, ...) {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof buf, fmt, ap);
        va_end(ap);
        err = buf;
        return s;
    }
};

namespace {

#define CU(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return w->fail(e_ == cudaErrorMemoryAllocation ? SPH_ERR_OOM : SPH_ERR_CUDA, "%s failed: %s (%s:%d)", #call, \
                           cudaGetErrorString(e_), __FILE__, __LINE__);                            \
    } while (0)
#define TRY(call)                          \
    do {                                   \
        sph_status s_ = (call);            \
        if (s_ != SPH_OK) return s_;       \
    } while (0)
#define LAUNCH(kern, n, threads, ...)                                                  \
    do {                                                                               \
        if ((n) > 0) {                                                                 \
            kern<<<cdiv((n), (threads)), (threads), 0, w->st>>>(__VA_ARGS__);           \
            w->launches++;                                                             \
        }                                                                              \
    } while (0)

inline uint32_t make_handle(size_t slot, uint32_t gen) { return (uint32_t)slot | (gen << 16); }
// slot of a live fluid / boundary handle, or -1
inline int fluid_slot(const sph_world* w, uint32_t handle) {
    const uint32_t slot = handle & 0xFFFFu;
    if (slot >= w->fluids.size() || !w->fluids[slot].alive || (w->fluids[slot].gen & 0xFFFFu) != (handle >> 16)) return -1;
    return (int)slot;
}
inline int boundary_slot(const sph_world* w, uint32_t handle) {
    const uint32_t slot = handle & 0xFFFFu;
    if (slot >= w->bounds.size() || !w->bounds[slot].alive || (w->bounds[slot].gen & 0xFFFFu) != (handle >> 16)) return -1;
    return (int)slot;
}
#define FLUID_OR_FAIL(var, handle)                                                                   \
    const int var##_slot_ = fluid_slot(w, handle);                                                   \
    if (var##_slot_ < 0) return w->fail(SPH_ERR_INVALID, "bad fluid handle %u", (unsigned)(handle)); \
    const uint32_t var = (uint32_t)var##_slot_;
#define BOUNDARY_OR_FAIL(var, handle)                                                                   \
    const int var##_slot_ = boundary_slot(w, handle);                                                   \
    if (var##_slot_ < 0) return w->fail(SPH_ERR_INVALID, "bad boundary handle %u", (unsigned)(handle)); \
    const uint32_t var = (uint32_t)var##_slot_;

enum { SP_DIV_EVAL = 0, SP_DIV_UPD, SP_PRED, SP_PUPD, SP_COUNT };
sph_status span_begin(sph_world* w, int slot) {
    if (w->cap) return SPH_OK;
    if (w->n_spans == w->spans.size()) {
        sph_world::Span s{slot, nullptr, nullptr};
        CU(cudaEventCreate(&s.a));
        CU(cudaEventCreate(&s.b));
        w->spans.push_back(s);
    }
    w->spans[w->n_spans].slot = slot;
    CU(cudaEventRecord(w->spans[w->n_spans].a, w->st));
    return SPH_OK;
}
sph_status span_end(sph_world* w) {
    if (w->cap) return SPH_OK;
    CU(cudaEventRecord(w->spans[w->n_spans].b, w->st));
    w->n_spans++;
    return SPH_OK;
}

// a phase boundary's timing event; a step graph records none (its conditional bodies cannot hold event nodes)
sph_status ev_record(sph_world* w, int e) {
    if (!w->cap) CU(cudaEventRecord(w->ev[e], w->st));
    return SPH_OK;
}

sph_status upload_consts(sph_world* w) {
    CU(cudaMemcpyToSymbolAsync(C, &w->hc, sizeof(Consts), 0, cudaMemcpyHostToDevice, w->st));
    g_const_owner = w;
    return SPH_OK;
}

sph_status enter(sph_world* w) {
    CU(cudaSetDevice(w->desc.device));
    if (g_const_owner != w) TRY(upload_consts(w));
    return SPH_OK;
}

void fill_static_consts(sph_world* w) {
    Consts& c = w->hc;
    c.h = w->h;
    c.inv_h = 1.0f / w->h;
    c.h2 = w->h * w->h;
    c.xysub = w->slab.active ? 1 : w->xysub;  // slab worlds cut x into cell columns of width h: plain cells there
    c.xysub_f = (float)c.xysub;
    c.h_reach = std::nextafter(w->h * 1.00001f, INFINITY);
    c.sigma = 8.0f / (3.14159265358979323846f * w->h * w->h * w->h);
    c.dsigma = c.sigma / w->h;
    c.dsigma6 = 6.0f * c.dsigma;
    c.kw = w->desc.kernel_density;
    c.kg = w->desc.kernel_gradient;
    c.kgen = (c.kw != 0 || c.kg != 0) ? 1 : 0;
    {
        const float h = w->h, pi = 3.14159265358979323846f;
        auto powi = [](float x, int n) { float r = 1.f; for (int k = 0; k < n; ++k) r *= x; return r; };
        c.poly6_n = (float)(315.0 / 64.0) / (pi * powi(h, 9));
        c.spiky_n = 15.0f / (pi * powi(h, 6));
        c.visc_n = 15.0f / (2.0f * pi * powi(h, 3));
    }
    {
        const double a = (double)F32_EPS * (double)F32_EPS, b = 1.0e-5 * (double)w->h * 1.0e-5 * (double)w->h;
        c.g_t2 = (float)std::max(a, b);
    }
    c.n_fluid = (uint32_t)w->Ntot;
    c.i_begin = w->own_begin;
    c.n_owned = (uint32_t)w->N;
    c.n_bound = (uint32_t)w->B;
    c.n_fluids = (int)w->fluids.size();
    c.n_bounds = (int)w->bounds.size();
    for (size_t f = 0; f < w->fluids.size(); ++f)
        c.fluids[f] = {w->fluids[f].density0, w->fluids[f].memberships, w->fluids[f].filter, w->fluids[f].uniform_mass};
    for (size_t b = 0; b < w->bounds.size(); ++b) c.bounds[b] = {w->bounds[b].memberships, w->bounds[b].filter};
    c.stride = w->stride;
    c.cap_f = w->lists.cap_f;
    c.cap_b = w->lists.cap_b;
}

// Raises the list capacities to at least cf / cb rows, grows the lists and refreshes the constants that carry the capacities.
sph_status grow_lists(sph_world* w, uint32_t cf, uint32_t cb) {
    ListState& L = w->lists;
    if (cf <= L.cap_f && cb <= L.cap_b) return SPH_OK;
    L.cap_f = std::max(L.cap_f, cf);
    L.cap_b = std::max(L.cap_b, cb);
    CU(L.ensure(0, w->stride));  // (the counts keep their size)
    fill_static_consts(w);
    return upload_consts(w);
}

// ---- exclusive scan over n u32 (in place) -------------------------------------------------------
sph_status scan_exclusive(sph_world* w, uint32_t* data, size_t n, int level = 0) {
    if (n == 0) return SPH_OK;
    uint32_t nb = cdiv(n, SCAN_B);
    if (nb == 1) {
        k_scan_block<<<1, SCAN_T, 0, w->st>>>(data, data, (uint32_t)n, nullptr);
        w->launches++;
        return SPH_OK;
    }
    if (level >= 3) return w->fail(SPH_ERR_INVALID, "scan too deep");
    CU(w->scan_aux[level].ensure(nb));
    k_scan_block<<<nb, SCAN_T, 0, w->st>>>(data, data, (uint32_t)n, w->scan_aux[level].p);
    w->launches++;
    TRY(scan_exclusive(w, w->scan_aux[level].p, nb, level + 1));
    k_scan_add<<<nb, SCAN_T, 0, w->st>>>(data, (uint32_t)n, w->scan_aux[level].p);
    w->launches++;
    return SPH_OK;
}

// K arrays of the same length scanned together (in place, exclusive); n <= 2048 * 2048 * 2048.  aux: three levels of block
// sums (default: the step's scan_aux_k)
template <int K>
sph_status scan_exclusive_k(sph_world* w, ScanSet<K> arrays, size_t n, int level = 0, DBuf<uint32_t>* aux = nullptr) {
    if (!aux) aux = w->scan_aux_k;
    if (n == 0) return SPH_OK;
    uint32_t nb = cdiv(n, SCAN_B);
    ScanSet<K> sums;
    for (int a = 0; a < K; ++a) sums.a[a] = nullptr;
    if (nb == 1) {
        k_scanK_block<K><<<1, SCAN_T, 0, w->st>>>(arrays, (uint32_t)n, sums);
        w->launches++;
        return SPH_OK;
    }
    if (level >= 3) return w->fail(SPH_ERR_INVALID, "scan too deep");
    CU(aux[level].ensure((size_t)K * nb));
    for (int a = 0; a < K; ++a) sums.a[a] = aux[level].p + (size_t)a * nb;
    k_scanK_block<K><<<nb, SCAN_T, 0, w->st>>>(arrays, (uint32_t)n, sums);
    w->launches++;
    TRY(scan_exclusive_k<K>(w, sums, nb, level + 1, aux));
    k_scanK_add<K><<<nb, SCAN_T, 0, w->st>>>(arrays, (uint32_t)n, sums);
    w->launches++;
    return SPH_OK;
}

// ---- sorted order <-> caller order (layout: sph_order.cuh) --------------------------------------------
// One column of an export: `src` read over the sorted slots [s0, s0 + n) (a null orig maps slot s to row s).  The caller
// rows [first, first + count) are copied to `host`; or, with `dev` set, every row is written straight into that device array.
template <class V>
struct Col {
    V src;
    const uint32_t* orig;
    uint32_t s0, n;
    size_t first, count;
    typename V::T* host;
    typename V::T* dev = nullptr;
};
// fluid rows, from the slots this GPU owns
template <class V>
Col<V> fluid_col(const sph_world* w, V src, size_t first, size_t count, typename V::T* host) {
    return {src, w->orig[w->cur].p, w->own_begin, (uint32_t)w->N, first, count, host};
}
// boundary rows, from every boundary slot
template <class V>
Col<V> boundary_col(const sph_world* w, V src, size_t first, size_t count, typename V::T* host) {
    return {src, w->borig[w->bcur].p, 0u, (uint32_t)w->B, first, count, host};
}

// At least `words` 4-byte words of rows_scratch.  It grows to the request exactly, without DBuf's headroom: a world never
// holds more of it than the largest single call needed (stage_up's 11 words per particle, or a wide debug read's 36).
// Every call that uses it is done with it when it returns: export_rows and import_rows end in a stream synchronise.
sph_status ensure_rows_scratch(sph_world* w, size_t words) {
    if (words > w->rows_scratch.cap) {
        w->rows_scratch.release();
        CU(w->rows_scratch.ensure(words));
    }
    return SPH_OK;
}

// Enqueues every column's export and host copy, each host column in a region of its own, then synchronises if any
// column went to the host.
template <class... V>
sph_status export_rows(sph_world* w, const Col<V>&... cols) {
    size_t words = 0;
    ((words += cols.dev ? 0 : cols.src.width * (size_t)cols.n), ...);
    const bool to_host = (!cols.dev || ...);
    TRY(ensure_rows_scratch(w, words));
    size_t at = 0;
    auto one = [&](const auto& col) -> sph_status {
        using View = std::decay_t<decltype(col.src)>;
        using T = typename View::T;
        static_assert(sizeof(T) == sizeof(uint32_t), "rows_scratch holds 4-byte values");
        T* dst = col.dev ? col.dev : reinterpret_cast<T*>(w->rows_scratch.p + at);
        LAUNCH(k_export<View>, col.n, 256, col.n, col.s0, col.orig, col.src, dst);
        if (col.dev) return SPH_OK;
        const size_t width = col.src.width;
        CU(cudaMemcpyAsync(col.host, dst + width * col.first, width * col.count * sizeof(T), cudaMemcpyDeviceToHost, w->st));
        at += width * col.n;
        return SPH_OK;
    };
    sph_status s = SPH_OK;
    if (!(((s = one(cols)) == SPH_OK) && ...)) return s;
    if (to_host) CU(cudaStreamSynchronize(w->st));
    return SPH_OK;
}

// The mirror: caller rows [first, first + count) from the host into the slots this GPU owns (k_import), then a stream
// synchronise.  Any source may be null; the velocity changes land in `vc` (a host force writes accelerations back there).
struct ImportRows {
    const float *pos = nullptr, *vel = nullptr, *vc = nullptr, *mass = nullptr;
    const uint32_t* fid = nullptr;
};
sph_status import_rows(sph_world* w, const ImportRows& in, size_t first, size_t count, float4* vc) {
    const void* src[5] = {in.pos, in.vel, in.vc, in.mass, in.fid};
    const size_t width[5] = {3, 3, 3, 1, 1};
    size_t words = 0;
    for (int a = 0; a < 5; ++a) words += src[a] ? width[a] * count : 0;
    TRY(ensure_rows_scratch(w, words));
    const void* dev[5] = {};
    size_t at = 0;
    for (int a = 0; a < 5; ++a)
        if (src[a]) {
            dev[a] = w->rows_scratch.p + at;
            CU(cudaMemcpyAsync(w->rows_scratch.p + at, src[a], width[a] * count * sizeof(uint32_t), cudaMemcpyHostToDevice, w->st));
            at += width[a] * count;
        }
    const int c = w->cur;
    auto f = [&](int a) { return static_cast<const float*>(dev[a]); };
    LAUNCH(k_import, w->N, 256, (uint32_t)w->N, w->own_begin, w->orig[c].p, f(0), f(1), f(2), f(3), static_cast<const uint32_t*>(dev[4]), w->pos[c].p,
           w->vel[c].p, vc, (uint32_t)first, (uint32_t)(first + count));
    CU(cudaStreamSynchronize(w->st));
    return SPH_OK;
}

// ---- host <-> device staging --------------------------------------------------------------------
// Device holds the truth -> pull everything back into the host vectors (original order).
sph_status stage_down(sph_world* w) {
    if (w->staged) return SPH_OK;
    size_t N = w->N;
    w->rows.resize(N);
    if (N) {
        // one column per call: the scratch holds 3 words per particle, not all 11
        const int c = w->cur;
        FluidRows& r = w->rows;
        TRY(export_rows(w, fluid_col(w, Xyz{w->pos[c].p}, 0, N, r.pos.data())));
        TRY(export_rows(w, fluid_col(w, Xyz{w->vel[c].p}, 0, N, r.vel.data())));
        TRY(export_rows(w, fluid_col(w, Xyz{w->vc[c].p}, 0, N, r.vc.data())));
        TRY(export_rows(w, fluid_col(w, U32<uint32_t>{w->gid[c].p}, 0, N, r.gid.data())));
        if (w->desc.solver == SPH_SOLVER_IISPH && w->press[c].p) TRY(export_rows(w, fluid_col(w, Rows<1>{w->press[c].p}, 0, N, r.press.data())));
    }
    w->staged = true;
    w->lists_valid = false;
    w->grid_ready = false;
    w->nb_valid = false;
    return SPH_OK;
}

void recompute_offsets(sph_world* w) {
    size_t o = 0;
    for (auto& f : w->fluids) {
        f.offset = o;
        o += f.n;
    }
    w->N = o;
    o = 0;
    for (auto& b : w->bounds) {
        b.offset = o;
        o += b.n;
    }
    w->B = o;
}

sph_status ensure_fluid_buffers(sph_world* w) {
    size_t N = std::max(w->Ntot, w->N);
    for (int k = 0; k < 2; ++k) {
        if (k == w->protect_buf) continue;
        bool keep = k == w->cur;  // the live buffers may be grown while they hold particles (ghost append)
        CU(w->pos[k].ensure(N, keep, w->st));
        CU(w->vel[k].ensure(N, keep, w->st));
        CU(w->vc[k].ensure(N, keep, w->st));
        CU(w->orig[k].ensure(N, keep, w->st));
        CU(w->gid[k].ensure(N, keep, w->st));
        if (w->desc.solver == SPH_SOLVER_IISPH) CU(w->press[k].ensure(N, keep, w->st));
    }
    CU(w->vs.ensure(N));
    CU(w->pvx4.ensure(N));
    CU(w->pk4.ensure(N));
    CU(w->vyz2.ensure(N));
    CU(w->acc.ensure(N));
    CU(w->dens.ensure(N + 8));
    CU(w->alpha.ensure(N + 8));
    CU(w->kappa.ensure(N + 8));
    CU(w->divv.ensure(N + 8));
    CU(w->pred.ensure(N + 8));
    CU(w->cid.ensure(N));
    CU(w->rank.ensure(N));
    CU(w->perm.ensure(N));
    if (w->desc.deterministic) CU(w->skey.ensure(N));
    w->stride = (uint32_t)((N + 31) / 32 * 32);
    CU(w->lists.ensure(N, w->stride));
    uint32_t nblk = cdiv(std::max<size_t>(N, 1), std::min(PASS_T, NBR_T));
    CU(w->partial.ensure((size_t)nblk * std::max<size_t>(1, w->fluids.size())));
    return SPH_OK;
}

// Host vectors hold the truth -> build the device state (sorted order starts as the identity).
sph_status stage_up(sph_world* w) {
    if (!w->staged) return SPH_OK;
    recompute_offsets(w);
    size_t N = w->N;
    w->Ntot = N;
    w->own_begin = 0;
    TRY(ensure_fluid_buffers(w));
    w->vol_all_default = true;
    if (N) {
        const std::vector<float>& vol = w->rows.vol;
        std::vector<float> mass(N);
        std::vector<uint32_t> fid(N);
        bool all_default = true;
        for (size_t g = 0; g < N; ++g) all_default = all_default && vol[g] == w->rows.vol0;
        w->vol_all_default = all_default;
        for (size_t f = 0; f < w->fluids.size(); ++f) {
            bool uniform = w->fluids[f].n > 0;
            for (size_t i = 0; i < w->fluids[f].n; ++i) {
                size_t g = w->fluids[f].offset + i;
                mass[g] = vol[g] * w->fluids[f].density0;  // fluid.rs:183-185
                fid[g] = (uint32_t)f;
                uniform = uniform && vol[g] == vol[w->fluids[f].offset];
            }
            w->fluids[f].uniform_mass = uniform ? mass[w->fluids[f].offset] : 0.f;
        }
        int c = w->cur;
        LAUNCH(k_iota, N, 256, (uint32_t)N, w->orig[c].p);
        CU(cudaMemcpyAsync(w->gid[c].p, w->rows.gid.data(), N * sizeof(uint32_t), cudaMemcpyHostToDevice, w->st));
        CU(cudaMemsetAsync(w->pos[c].p, 0, N * sizeof(float4), w->st));
        CU(cudaMemsetAsync(w->vel[c].p, 0, N * sizeof(float4), w->st));
        if (w->desc.solver == SPH_SOLVER_IISPH)
            CU(cudaMemcpyAsync(w->press[c].p, w->rows.press.data(), N * sizeof(float), cudaMemcpyHostToDevice, w->st));
        // synchronises before the host temporaries go out of scope
        TRY(import_rows(w, {w->rows.pos.data(), w->rows.vel.data(), w->rows.vc.data(), mass.data(), fid.data()}, 0, N, w->vc[c].p));
    }
    w->staged = false;
    w->lists_valid = false;
    w->slab.global_valid = false;
    // a slab world takes the fast path on every rank or on none: volumes default to uniform there, and an empty
    // slab inherits the constant from its first immigrant only through the classic path -> keep it simple: require
    // particles with uniform volumes on this rank, otherwise fall back (all ranks are built by the same host code).
    w->unimass = w->desc.solver == SPH_SOLVER_DFSPH && w->fluids.size() == 1 && w->fluids[0].uniform_mass > 0.f;
    return SPH_OK;
}

sph_status upload_boundaries(sph_world* w) {
    if (!w->b_dirty) return SPH_OK;
    recompute_offsets(w);
    size_t B = w->B;
    for (int k = 0; k < 2; ++k) {
        CU(w->bpos[k].ensure(B));
        CU(w->bvel[k].ensure(B));
        CU(w->borig[k].ensure(B));
    }
    CU(w->bvol.ensure(B));
    CU(w->bcid.ensure(B));
    CU(w->brank.ensure(B));
    CU(w->bperm.ensure(B));
    CU(w->bforce.ensure(3 * B));
    w->b_box = CELL_BOX_EMPTY;
    for (size_t g = 0; g < B; ++g) cell_box_add(w->b_box, w->brows.pos[3 * g], w->brows.pos[3 * g + 1], w->brows.pos[3 * g + 2], w->h);
    if (B) {
        std::vector<float4> p(B), v(B);
        for (size_t b = 0; b < w->bounds.size(); ++b)
            for (size_t i = 0; i < w->bounds[b].n; ++i) {
                size_t g = w->bounds[b].offset + i;
                p[g] = make_float4(w->brows.pos[3 * g], w->brows.pos[3 * g + 1], w->brows.pos[3 * g + 2], 0.f);
                v[g] = make_float4(w->brows.vel[3 * g], w->brows.vel[3 * g + 1], w->brows.vel[3 * g + 2], __uint_as_float_host((uint32_t)b));
            }
        int c = w->bcur;
        CU(cudaMemcpyAsync(w->bpos[c].p, p.data(), B * sizeof(float4), cudaMemcpyHostToDevice, w->st));
        CU(cudaMemcpyAsync(w->bvel[c].p, v.data(), B * sizeof(float4), cudaMemcpyHostToDevice, w->st));
        LAUNCH(k_iota, B, 256, (uint32_t)B, w->borig[c].p);
        CU(cudaStreamSynchronize(w->st));
    }
    w->b_dirty = false;
    w->b_sorted_valid = false;
    w->lists_valid = false;
    return SPH_OK;
}

// Colliders keep their boundaries on the device; before the host copy is edited or handed out, bring it up to date.
sph_status pull_boundaries(sph_world* w) {
    if (!w->hb_stale) return SPH_OK;
    TRY(enter(w));
    const size_t B = w->B;
    const int bc = w->bcur;
    TRY(export_rows(w, boundary_col(w, Xyz{w->bpos[bc].p}, 0, B, w->brows.pos.data()), boundary_col(w, Xyz{w->bvel[bc].p}, 0, B, w->brows.vel.data())));
    w->hb_stale = false;
    return SPH_OK;
}

// fluid.rs:88-98 apply_particles_removal (+ solver scratch filtering dfsph_solver.rs:550-559)
sph_status apply_pending_deletes(sph_world* w) {
    bool any = false;
    for (auto& f : w->fluids) any |= f.n_pending != 0;
    if (!any) return SPH_OK;
    TRY(stage_down(w));
    std::vector<uint8_t> keep;
    keep.reserve(w->N);
    for (auto& f : w->fluids) {
        size_t kept = 0;
        for (size_t i = 0; i < f.n; ++i) {
            keep.push_back(!(f.n_pending && f.pending_delete[i]));
            kept += keep.back();
        }
        f.n = kept;
        f.pending_delete.assign(kept, 0);
        f.n_pending = 0;
    }
    w->rows.keep(keep);
    recompute_offsets(w);
    return SPH_OK;
}

// ---- step phases ----------------------------------------------------------------------------------
// Where a StepScalars field begins and ends, in bytes: the bounds of a reset or a read-back
#define SS_BEGIN(f) offsetof(StepScalars, f)
#define SS_END(f) (offsetof(StepScalars, f) + sizeof(StepScalars::f))

// Enqueues the copy of the StepScalars bytes [from, to) into the pinned mirror; the caller synchronises before reading it
sph_status read_scalars(sph_world* w, size_t from, size_t to) {
    CU(cudaMemcpyAsync(reinterpret_cast<char*>(w->h_ss) + from, reinterpret_cast<const char*>(w->d_ss.p) + from, to - from,
                       cudaMemcpyDeviceToHost, w->st));
    return SPH_OK;
}

// The dense cell grid over the fluid's cell box, with the boundaries' box and one padding cell each side: its constants
// (uploaded) and cell arrays.  *ncell: its cells.
sph_status grid_size(sph_world* w, const CellBox& fluid, size_t* ncell_out) {
    CellBox hb = fluid;
    merge(hb, w->b_box);  // boundary box: static, kept on the host
    long long dims[3];
    for (int a = 0; a < 3; ++a) dims[a] = (long long)hb.hi[a] - hb.lo[a] + 3;  // one padding cell each side
    double ncell_d = (double)dims[0] * (double)dims[1] * (double)dims[2];
    if (ncell_d > 1.0e9) return w->fail(SPH_ERR_OOM, "dense cell grid too large: %lld x %lld x %lld cells of width h", dims[0], dims[1], dims[2]);
    const int xys = w->slab.active ? 1 : w->xysub;  // x / y bins per cell (row order, Consts::xysub)
    if (ncell_d * xys * xys > 2.0e9) return w->fail(SPH_ERR_OOM, "dense cell grid too large: %lld x %lld x %lld cells of width h", dims[0], dims[1], dims[2]);
    size_t ncell = (size_t)dims[0] * dims[1] * dims[2] * xys * xys;
    w->hc.ox = (hb.lo[0] - 1) * xys;
    w->hc.oy = (hb.lo[1] - 1) * xys;
    w->hc.oz = hb.lo[2] - 1;
    w->hc.nx = (int)dims[0] * xys;
    w->hc.ny = (int)dims[1] * xys;
    w->hc.nz = (int)dims[2];
    fill_static_consts(w);
    TRY(upload_consts(w));
    CU(w->cstart.ensure(ncell + 1));
    CU(w->bstart.ensure(ncell + 1));
    w->stats.grid_dims[0] = (uint32_t)dims[0];
    w->stats.grid_dims[1] = (uint32_t)dims[1];
    w->stats.grid_dims[2] = (uint32_t)dims[2];
    *ncell_out = ncell;
    return SPH_OK;
}

// The boundaries' counting sort on the current grid — reused while neither the boundaries nor the cell mapping changed
// (static tanks).  ncell: the grid's cells.
sph_status sort_boundaries(sph_world* w, size_t ncell) {
    const size_t B = w->B;
    const int bc = w->bcur;
    const int xys = w->slab.active ? 1 : w->xysub;
    const int gridkey[6] = {w->hc.ox, w->hc.oy, w->hc.oz, w->hc.nx, w->hc.ny, w->hc.nz};
    const bool reuse_b = w->b_sorted_valid && memcmp(gridkey, w->b_sorted_grid, sizeof gridkey) == 0;
    w->b_reused = reuse_b;
    if (!reuse_b) CU(cudaMemsetAsync(w->bstart.p, 0, (ncell + 1) * sizeof(uint32_t), w->st));
    if (B && !reuse_b) {
        if (xys > 1) LAUNCH(k_cell_hist_xy, B, 256, w->bpos[bc].p, (uint32_t)B, w->bcid.p, w->brank.p, w->bstart.p);
        else LAUNCH(k_cell_hist, B, 256, w->bpos[bc].p, (uint32_t)B, w->bcid.p, w->brank.p, w->bstart.p, (const uint32_t*)nullptr, 0u);
        TRY(scan_exclusive(w, w->bstart.p, ncell + 1));
        // in-cell order by original index: the same whether the input is a fresh upload or the last sort of boundaries that
        // colliders moved on the device
        const bool det = w->desc.deterministic;
        if (det) CU(w->skey.ensure(B));
        LAUNCH(k_cell_scatter, B, 256, (uint32_t)B, w->bcid.p, w->brank.p, w->bstart.p, w->bperm.p, (const uint32_t*)w->borig[bc].p,
               (const float4*)nullptr, det ? w->skey.p : nullptr);
        if (det) LAUNCH(k_cell_sort, ncell, 256, (uint32_t)ncell, w->bstart.p, w->bperm.p, w->skey.p);
        GatherSet g;
        memset(&g, 0, sizeof g);
        g.in4[0] = w->bpos[bc].p; g.out4[0] = w->bpos[bc ^ 1].p;
        g.in4[1] = w->bvel[bc].p; g.out4[1] = w->bvel[bc ^ 1].p;
        g.n4 = 2;
        g.in1[0] = w->borig[bc].p; g.out1[0] = w->borig[bc ^ 1].p;
        g.n1 = 1;
        LAUNCH(k_gather, B, 256, (uint32_t)B, w->bperm.p, g);
        w->bcur = bc ^ 1;
    }
    if (!reuse_b) {
        memcpy(w->b_sorted_grid, gridkey, sizeof gridkey);
        w->b_sorted_valid = true;
    }
    return SPH_OK;
}

sph_status phase_grid(sph_world* w) {
    size_t N = w->Ntot;  // the sort covers owned + ghost slots
    int c = w->cur;
    // slab worlds: the prologue appended immigrants / ghosts behind the owned range of the live arrays and flagged the
    // particles that left; the sort reads [off, off + Nin) and drops the flagged slots.  Elsewhere: all N slots from 0.
    const uint32_t off = w->slab.active ? w->slab.sort_off : 0u;
    const size_t Nin = w->slab.active ? w->slab.sort_n : N;
    const uint32_t* dead = w->slab.active ? w->slab.flag.p : nullptr;
    const uint32_t n_dead = w->slab.active ? w->slab.sort_dead_n : 0u;
    size_t ncell;
    if (w->cap) {  // a step graph runs on the envelope's grid, which graph_prepare set up
        CU(cudaMemsetAsync(reinterpret_cast<char*>(w->d_ss.p) + SS_BEGIN(err), 0, SS_END(contacts_f) - SS_BEGIN(err), w->st));
        ncell = (size_t)w->hc.nx * w->hc.ny * w->hc.nz;
    } else {
        StepScalars init{};
        init.grid = CELL_BOX_EMPTY;
        CU(cudaMemcpyAsync(w->d_ss.p, &init, SS_END(contacts_f), cudaMemcpyHostToDevice, w->st));
        CellBox hb;
        if (w->nb_valid && !w->slab.active && N) {
            // positions are exactly what the last step's k_update_positions wrote (no host edit since): its bounds came back with
            // that step's final read-back, so this step starts without a bounds pass and without a host round trip
            hb = w->nb;
        } else {
            if (Nin) {
                k_bounds<<<std::min<uint32_t>(cdiv(Nin, 256), 296), 256, 0, w->st>>>(w->pos[c].p + off, (uint32_t)Nin, &w->d_ss.p->grid);
                w->launches++;
            }
            TRY(read_scalars(w, SS_BEGIN(grid), SS_END(grid)));
            CU(cudaStreamSynchronize(w->st));
            hb = w->h_ss->grid;
        }
        w->nb_valid = false;
        if (hb.bad || w->b_box.bad) return w->fail(SPH_ERR_INVALID, "non-finite or out-of-range particle coordinates");
        TRY(grid_size(w, hb, &ncell));
    }
    const int xys = w->slab.active ? 1 : w->xysub;  // x / y bins per cell (row order, Consts::xysub)
    // fluid: counting sort by cell, then reorder every persistent array
    CU(cudaMemsetAsync(w->cstart.p, 0, (ncell + 1) * sizeof(uint32_t), w->st));
    if (xys > 1) LAUNCH(k_cell_hist_xy, Nin, 256, w->pos[c].p + off, (uint32_t)Nin, w->cid.p, w->rank.p, w->cstart.p);  // (never a slab world: no dead slots)
    else LAUNCH(k_cell_hist, Nin, 256, w->pos[c].p + off, (uint32_t)Nin, w->cid.p, w->rank.p, w->cstart.p, dead, n_dead);
    TRY(scan_exclusive(w, w->cstart.p, ncell + 1));
    const bool det = w->desc.deterministic;
    if (det) CU(w->skey.ensure(Nin));  // (a step graph's envelope allocated it: no allocation in capture)
    LAUNCH(k_cell_scatter, Nin, 256, (uint32_t)Nin, w->cid.p, w->rank.p, w->cstart.p, w->perm.p, (const uint32_t*)w->gid[c].p + off,
           w->fluids.size() > 1 ? (const float4*)w->vel[c].p + off : (const float4*)nullptr, det ? w->skey.p : nullptr);
    if (det) LAUNCH(k_cell_sort, ncell, 256, (uint32_t)ncell, w->cstart.p, w->perm.p, w->skey.p);
    if (N) {
        GatherSet g;
        memset(&g, 0, sizeof g);
        g.in4[0] = w->pos[c].p + off; g.out4[0] = w->pos[c ^ 1].p;
        g.in4[1] = w->vel[c].p + off; g.out4[1] = w->vel[c ^ 1].p;
        g.in4[2] = w->vc[c].p + off;  g.out4[2] = w->vc[c ^ 1].p;
        g.n4 = 3;
        g.in1[0] = w->orig[c].p + off; g.out1[0] = w->orig[c ^ 1].p;  // (slab worlds overwrite orig with the identity after the sort)
        g.in1[1] = w->gid[c].p + off; g.out1[1] = w->gid[c ^ 1].p;
        g.n1 = 2;
        if (w->desc.solver == SPH_SOLVER_IISPH) {
            g.in1[2] = reinterpret_cast<const uint32_t*>(w->press[c].p);
            g.out1[2] = reinterpret_cast<uint32_t*>(w->press[c ^ 1].p);
            g.n1 = 3;
        }
        // reorder + v* = vel + vc (the divergence solve works on vel + vc carried over from the previous step, Appendix A.3.2) in one pass
        LAUNCH(k_gather_vstar, N, 256, (uint32_t)N, w->perm.p, g, w->vs.p, w->unimass ? w->pvx4.p : nullptr, w->unimass ? w->vyz2.p : nullptr);
        w->cur = c ^ 1;
    }
    TRY(sort_boundaries(w, ncell));
    if (w->cap && !w->b_reused) return w->fail(SPH_ERR_INVALID, "step graph: the boundaries are not sorted on the envelope's grid");
    CU(cudaGetLastError());
    if (w->slab.active) {
        TRY(slab_after_sort(w));
        fill_static_consts(w);
        TRY(upload_consts(w));
    }
    return SPH_OK;
}

// Inputs and outputs of the density sweep that the DFSPH neighbour search runs over its fresh lists (density_alpha_div)
sph_status density_args(sph_world* w, DensArgs* D) {
    if (w->unimass) {
        CU(w->tex_vyz.bind(w->vyz2));
        CU(w->tex_pvx.bind(w->pvx4));
    } else {
        CU(w->tex_vs.bind(w->vs));
    }
    *D = DensArgs{w->unimass ? w->pvx4.p : w->pos[w->cur].p, w->unimass ? w->tex_pvx.obj : 0, w->vs.p, w->unimass ? 0 : w->tex_vs.obj, w->vyz2.p,
                  w->unimass ? w->tex_vyz.obj : 0, w->dens.p, w->alpha.p, w->divv.p, w->kappa.p, w->pk4.p, w->partial.p, &w->d_ss.p->err};
    return SPH_OK;
}

// `speculative` (optional) enqueues the work that follows the neighbour search and only writes scratch (the density
// pass): it is launched BEFORE the host learns whether the lists overflowed, so the GPU is busy during that round trip;
// on overflow the lists are rebuilt with a larger capacity and the speculative work is simply enqueued again.
// With DFSPH the search itself computes rho, alpha and the first divergence evaluation (density_alpha_div); on overflow the
// relaunched search computes them again.
sph_status phase_neighbors(sph_world* w, sph_status (*speculative)(sph_world*) = nullptr) {
    size_t N = w->N, B = w->B;
    int c = w->cur, bc = w->bcur;
    const bool multi = w->fluids.size() > 1;
    const bool dens = N && w->desc.solver == SPH_SOLVER_DFSPH, uni = dens && w->unimass;
    DensArgs D{};
    if (dens) TRY(density_args(w, &D));
    using NbrKernel = void (*)(const float4*, const float4*, const uint32_t*, const float4*, const float4*, const uint32_t*, ListsOut,
                               uint32_t*, DensArgs);
    NbrKernel search;
    if (w->hc.xysub > 1) {  // row order
        if (multi) search = dens ? k_neighbors_xy<true, true, false> : k_neighbors_xy<true, false, false>;
        else if (dens) search = uni ? k_neighbors_xy<false, true, true> : k_neighbors_xy<false, true, false>;
        else search = k_neighbors_xy<false, false, false>;
    } else {
        if (multi) search = dens ? k_neighbors<true, true, false> : k_neighbors<true, false, false>;
        else if (dens) search = uni ? k_neighbors<false, true, true> : k_neighbors<false, true, false>;
        else search = k_neighbors<false, false, false>;
    }
    if (B) {  // compute_boundary_volumes dfsph_solver.rs:72-96: the reference recomputes them every substep; they only
              // depend on the boundary positions, so they are reused while the boundaries are unchanged
        if (!w->b_reused) {
            StepScalars* ss = w->d_ss.p;
            if (w->hc.xysub > 1) LAUNCH(k_boundary_volumes_xy, B, 128, w->bpos[bc].p, w->bvel[bc].p, w->bstart.p, w->bvol.p, &ss->contacts_bb, &ss->err);
            else LAUNCH(k_boundary_volumes, B, 128, w->bpos[bc].p, w->bvel[bc].p, w->bstart.p, w->bvol.p, &ss->contacts_bb, &ss->err);
            LAUNCH(k_set_w, B, 256, (uint32_t)B, w->bpos[bc].p, w->bvol.p);
        }
        for (auto& b : w->bounds)
            if (b.want_forces) {
                CU(cudaMemsetAsync(w->bforce.p, 0, 3 * B * sizeof(float), w->st));
                break;
            }
    }
    for (int attempt = 0; attempt < 8 && N; ++attempt) {
        CU(cudaMemsetAsync(w->d_ss.p->max_nb, 0, sizeof(StepScalars::max_nb), w->st));
        LAUNCH(search, N, NBR_T, w->pos[c].p, w->vel[c].p, w->cstart.p, w->bpos[bc].p, w->bvel[bc].p, w->bstart.p, w->lists.out(), w->d_ss.p->max_nb, D);
        if (w->cap) {  // a step graph checks the capacities on the device and skips the rest of the step past them
            k_lists_check<<<1, 1, 0, w->st>>>(w->graphs.ctl.p, w->graphs.rec.p, w->d_ss.p, w->lists.cap_f, w->lists.cap_b, w->graphs.h_lists);
            break;
        }
        TRY(read_scalars(w, SS_BEGIN(err), SS_END(max_nb)));  // pinned: the copy is truly asynchronous
        CU(cudaEventRecord(w->ev_lists, w->st));
        CU(cudaEventRecord(w->ev[EV_NBR], w->st));
        if (speculative) TRY(speculative(w));
        CU(cudaEventSynchronize(w->ev_lists));
        const StepScalars& S = *w->h_ss;
        // (a zero density of the search's own density sweep is reported with the other zero densities at the end of the step)
        if (S.err & ~ERR_SEARCH_ZERO_DENSITY)
            return w->fail(SPH_ERR_ZERO_DENSITY, "zero boundary-volume denominator (reference assert dfsph_solver.rs:92)");
        w->stats.max_neighbors = S.max_nb[0];
        w->max_nb_b = S.max_nb[1];
        if (S.max_nb[0] <= w->lists.cap_f && S.max_nb[1] <= w->lists.cap_b) break;
        if (speculative) CU(cudaMemsetAsync(&w->d_ss.p->err, 0, sizeof(int), w->st));  // error word of the discarded density pass or sweep
        TRY(grow_lists(w, (S.max_nb[0] + 15) / 16 * 16, (S.max_nb[1] + 15) / 16 * 16));
    }
    if (!N) {  // boundaries only
        TRY(ev_record(w, EV_NBR));
        if (speculative) TRY(speculative(w));
    }
    if (N) {
        k_sum_u32<<<std::min<uint32_t>(cdiv(N, 256), 1184), 256, 0, w->st>>>((uint32_t)N, w->lists.cnt_f.p + w->own_begin, w->lists.cnt_b.p + w->own_begin,
                                                                             &w->d_ss.p->contacts_f);
        w->launches++;
    }
    if (dens) w->fused_nblk = cdiv(N, NBR_T);  // one error partial per block, summed by read_error()
    CU(cudaGetLastError());
    w->lists_valid = true;
    if (speculative) TRY(post_density_refresh(w));
    return SPH_OK;
}

// the particle count of every fluid as the loop error divides by it (slab worlds: over all ranks)
std::array<float, MAX_FLUIDS> loop_sizes(const sph_world* w) {
    std::array<float, MAX_FLUIDS> n{};
    for (size_t f = 0; f < w->fluids.size() && f < (size_t)MAX_FLUIDS; ++f)
        n[f] = (float)(w->slab.active ? (double)w->slab.global_n : (double)w->fluids[f].n);
    return n;
}

// dfsph_step's loop bounds and exit rule for the divergence (true) or the pressure loop
LoopRule loop_rule(const sph_world* w, bool divergence) {
    LoopRule r;
    memset(&r, 0, sizeof r);
    const int force = divergence ? w->force_div : w->force_press;
    r.force = force;
    r.maxit = force >= 0 ? (uint32_t)force + 1 : (divergence ? w->desc.max_divergence_iter : w->desc.max_pressure_iter);
    r.min_iter = divergence ? w->desc.min_divergence_iter : w->desc.min_pressure_iter;
    r.max_error = divergence ? w->desc.max_divergence_error : w->desc.max_density_error;
    r.inv_dt = w->inv_dt;
    r.divergence = divergence;
    r.nf = (int)w->fluids.size();
    const std::array<float, MAX_FLUIDS> n = loop_sizes(w);
    memcpy(r.n, n.data(), sizeof r.n);
    return r;
}

// mean-per-fluid -> max over fluids (dfsph_solver.rs:153-158, :347-352)
sph_status read_error(sph_world* w, uint32_t nblk, float* out) {
    int nf = (int)w->fluids.size();
    k_reduce_partials<<<nf, 256, 0, w->st>>>(w->partial.p, nblk, nf, w->d_ss.p->loop_err);
    w->launches++;
    TRY(slab_allreduce(w, w->d_ss.p->loop_err, nf));  // multi-GPU: the means are over ALL ranks' particles
    TRY(read_scalars(w, SS_BEGIN(loop_err), SS_BEGIN(loop_err) + nf * sizeof(float)));
    CU(cudaStreamSynchronize(w->st));
    *out = loop_error(w->h_ss->loop_err, loop_sizes(w).data(), nf);
    return SPH_OK;
}

// A host loop's decision after evaluation i: loop_decision, with read_error (of nblk partials) into *err where it reads
sph_status host_decision(sph_world* w, const LoopRule& r, uint32_t i, uint32_t nblk, float* err, LoopDecision* d) {
    sph_status s = SPH_OK;
    *d = loop_decision(r, i, [&] {
        s = read_error(w, nblk, err);
        return *err;
    });
    return s;
}

bool any_bforce(const sph_world* w) {
    for (auto& b : w->bounds)
        if (b.want_forces) return true;
    return false;
}

#define DISPATCH2(kern, multi, bf, n, threads, ...)                                   \
    do {                                                                              \
        if (multi) {                                                                  \
            if (bf) LAUNCH((kern<true, true>), n, threads, __VA_ARGS__);              \
            else LAUNCH((kern<true, false>), n, threads, __VA_ARGS__);                \
        } else {                                                                      \
            if (bf) LAUNCH((kern<false, true>), n, threads, __VA_ARGS__);             \
            else LAUNCH((kern<false, false>), n, threads, __VA_ARGS__);               \
        }                                                                             \
    } while (0)
#define DISPATCH3(kern, b0, b1, b2, n, threads, ...)                                                                    \
    do {                                                                                                                 \
        if (b0) {                                                                                                        \
            if (b1) { if (b2) LAUNCH((kern<true, true, true>), n, threads, __VA_ARGS__); else LAUNCH((kern<true, true, false>), n, threads, __VA_ARGS__); } \
            else    { if (b2) LAUNCH((kern<true, false, true>), n, threads, __VA_ARGS__); else LAUNCH((kern<true, false, false>), n, threads, __VA_ARGS__); } \
        } else {                                                                                                         \
            if (b1) { if (b2) LAUNCH((kern<false, true, true>), n, threads, __VA_ARGS__); else LAUNCH((kern<false, true, false>), n, threads, __VA_ARGS__); } \
            else    { if (b2) LAUNCH((kern<false, false, true>), n, threads, __VA_ARGS__); else LAUNCH((kern<false, false, false>), n, threads, __VA_ARGS__); } \
        }                                                                                                                \
    } while (0)
#define DISPATCH1(kern, multi, n, threads, ...)                         \
    do {                                                                \
        if (multi) LAUNCH((kern<true>), n, threads, __VA_ARGS__);       \
        else LAUNCH((kern<false>), n, threads, __VA_ARGS__);            \
    } while (0)

// ---- gather passes: one wrapper per reference function ------------------------------------

// ghost refresh of v* in whichever representation the evaluations and the velocity fold (vel = v* for ghosts too) read:
// the packed records on the uniform-mass path (one NCCL group), else vs
sph_status refresh_vstar(sph_world* w) {
    if (!w->slab.active) return SPH_OK;
    if (w->unimass) {
        SlabArray a[2] = {{w->pvx4.p, sizeof(float4)}, {w->vyz2.p, sizeof(float2)}};
        return slab_refresh_n(w, a, 2);
    }
    return slab_refresh(w, w->vs.p, sizeof(float4));
}
// ghost refresh of the evaluation's output (kappa) — only needed when an update follows
sph_status refresh_kappa(sph_world* w) {
    if (!w->slab.active) return SPH_OK;
    if (w->unimass) return slab_refresh(w, w->pk4.p, sizeof(float4));
    return slab_refresh(w, w->kappa.p, sizeof(float));
}

sph_status launch_density_alpha(sph_world* w) {
    size_t N = w->N;
    int c = w->cur, bc = w->bcur;
    const bool multi = w->fluids.size() > 1;
    const Lists L = w->lists.view();
    DISPATCH1(k_density_alpha, multi, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, L, w->dens.p, w->alpha.p, &w->d_ss.p->err);
    return SPH_OK;  // the ghost refresh of rho follows in post_density_refresh(), once the list-capacity check has passed
}
// Ghost refresh of what the density pass produced (rho; DFSPH: also kappa of the fused first divergence evaluation).  Kept out
// of the density launch itself so that the launch stays purely local: it is enqueued SPECULATIVELY behind the neighbour
// search (before the host knows whether the lists overflowed), and a rank that has to regrow its lists and repeat it must not
// leave its neighbours waiting in a collective they entered once and it enters twice.
sph_status post_density_refresh(sph_world* w) {
    if (!w->slab.active || !w->N) return SPH_OK;
    if (w->desc.solver == SPH_SOLVER_DFSPH) {
        SlabArray a[2] = {{w->dens.p, sizeof(float)}, {w->unimass ? (void*)w->pk4.p : (void*)w->kappa.p, w->unimass ? sizeof(float4) : sizeof(float)}};
        return slab_refresh_n(w, a, 2);
    }
    return slab_refresh(w, w->dens.p, sizeof(float));  // XSPH / artificial viscosity / Akinci gather rho_j of ghosts
}
// compute_divergences (predict = false) / compute_predicted_densities (predict = true); returns #partials.
// The fluid term of the FIRST force of a single-fluid DFSPH world can ride with the divergence evaluations when it is an
// XSPHViscosity without a boundary term (see k_vel_divergence_xsph_u).
bool xsph_fusable(const sph_world* w) {
    if (w->desc.solver != SPH_SOLVER_DFSPH || !w->unimass || w->slab.active) return false;
    if (w->fluids.size() != 1 || w->fluids[0].forces.empty()) return false;
    const sph_force_desc& d = w->fluids[0].forces[0].d;
    return d.kind == SPH_FORCE_XSPH_VISCOSITY && d.p[0] != 0.f && (d.p[1] == 0.f || w->B == 0);
}
// ... and an Akinci2013SurfaceTension: its normals ride with the loop's first update (k_vel_update_u<.., NORMALS>) and its fluid
// term with the evaluation after it (k_vel_divergence_xsph_u<2>), when it is the first force of the single uniform-mass fluid
// and has no boundary term (no adhesion, or no boundaries) and no boundary wants forces.  Otherwise phase_forces computes it.
bool akinci_fusable_u(const sph_world* w) {
    if (w->desc.solver != SPH_SOLVER_DFSPH || !w->unimass || w->slab.active) return false;
    if (w->fluids.size() != 1 || w->fluids[0].forces.empty()) return false;
    const sph_force_desc& d = w->fluids[0].forces[0].d;
    return d.kind == SPH_FORCE_AKINCI2013_TENSION && d.p[0] != 0.f && (d.p[1] == 0.f || w->B == 0) && !any_bforce(w);
}
// Akinci2013 kernel-normalisation constants of `h` (akinci2013_surface_tension.rs): cohesion, its h^6 / 64 offset, adhesion
struct AkinciNorms {
    float coh_norm, h6_64, adh_norm;
};
AkinciNorms akinci_norms(float h) {
    return {32.0f / (3.14159265358979323846f * powf(h, 9.f)), powf(h, 6.f) / 64.0f, 0.007f / powf(h, 3.25f)};
}

// akinci: the Akinci fluid force rides along (evaluation 1 of the divergence loop, on the normals update 0 wrote).
sph_status launch_vel_divergence(sph_world* w, bool predict, uint32_t* nblk, bool akinci = false) {
    int c = w->cur, bc = w->bcur;
    const bool multi = w->fluids.size() > 1;
    const bool xsf = !predict && xsph_fusable(w), akf = !predict && akinci;
    if (xsf || akf) CU(w->xs.ensure(std::max(w->Ntot, w->N)));
    const Lists L = w->lists.view();
    if (w->unimass) {
        CU(w->tex_pvx.bind(w->pvx4));
        CU(w->tex_vyz.bind(w->vyz2));
    } else {
        CU(w->tex_vs.bind(w->vs));
    }
    float* out = predict ? w->pred.p : w->divv.p;
    const size_t N = w->N;
    if (w->unimass) {
        if (predict) {
            LAUNCH((k_vel_divergence_u<true>), N, PASS_T, w->pvx4.p, w->tex_pvx.obj, w->vyz2.p, w->tex_vyz.obj, w->bpos[bc].p, w->bvel[bc].p, L,
                   w->dens.p, w->alpha.p, out, w->pk4.p, w->partial.p, w->dt, &w->d_ss.p->err);
        } else if (xsf) {
            const float cf = w->fluids[0].forces[0].d.p[0];
            LAUNCH((k_vel_divergence_xsph_u<1>), N, PASS_T, w->pvx4.p, w->tex_pvx.obj, w->vyz2.p, w->tex_vyz.obj, w->bpos[bc].p, L, w->dens.p,
                   w->alpha.p, out, w->pk4.p, w->partial.p, w->xs.p, cf, (const float4*)nullptr, 0.f, 0.f);
        } else if (akf) {  // the Akinci fluid force rides along: xs = its sum, on the normals the update wrote
            const AkinciNorms an = akinci_norms(w->h);
            LAUNCH((k_vel_divergence_xsph_u<2>), N, PASS_T, w->pvx4.p, w->tex_pvx.obj, w->vyz2.p, w->tex_vyz.obj, w->bpos[bc].p, L, w->dens.p,
                   w->alpha.p, out, w->pk4.p, w->partial.p, w->xs.p, w->fluids[0].forces[0].d.p[0], w->normals.p, an.coh_norm, an.h6_64);
        } else {
            LAUNCH((k_vel_divergence_u<false>), N, PASS_T, w->pvx4.p, w->tex_pvx.obj, w->vyz2.p, w->tex_vyz.obj, w->bpos[bc].p, w->bvel[bc].p, L,
                   w->dens.p, w->alpha.p, out, w->pk4.p, w->partial.p, w->dt, &w->d_ss.p->err);
        }
    } else {
        DISPATCH2(k_vel_divergence, multi, predict, N, PASS_T, w->pos[c].p, w->vs.p, w->tex_vs.obj, w->vel[c].p, w->bpos[bc].p, w->bvel[bc].p, L,
                  w->dens.p, w->alpha.p, out, w->kappa.p, w->partial.p, w->dt, &w->d_ss.p->err);
    }
    *nblk = cdiv(N, PASS_T);
    return SPH_OK;
}
// compute_velocity_changes_for_divergence (pressure = false) / compute_velocity_changes (pressure = true).
// normals: the Akinci normals ride along (see akinci_fusable_u).
sph_status launch_vel_update(sph_world* w, bool pressure, bool normals = false) {
    int c = w->cur, bc = w->bcur;
    const bool multi = w->fluids.size() > 1, bf = any_bforce(w);
    const Lists L = w->lists.view();
    if (w->unimass) CU(w->tex_pk.bind(w->pk4));
    if (normals) CU(w->normals.ensure(std::max(w->Ntot, w->N)));
    const size_t N = w->N;
    if (normals)  // akinci_fusable_u: uniform mass, no boundary forces
        LAUNCH((k_vel_update_u<false, false, true>), N, PASS_T, w->pk4.p, w->tex_pk.obj, w->vel[c].p, w->bpos[bc].p, L, w->vc[c].p, w->pvx4.p,
               w->vyz2.p, w->bforce.p, w->inv_dt, w->dens.p, w->normals.p);
    else if (w->unimass)
        DISPATCH2(k_vel_update_u, bf, pressure, N, PASS_T, w->pk4.p, w->tex_pk.obj, w->vel[c].p, w->bpos[bc].p, L, w->vc[c].p, w->pvx4.p,
                  w->vyz2.p, w->bforce.p, w->inv_dt, (const float*)nullptr, (float4*)nullptr);
    else
        DISPATCH3(k_vel_update, multi, bf, pressure, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, L, w->kappa.p, w->vc[c].p, w->vs.p,
                  w->bforce.p, w->inv_dt);
    return refresh_vstar(w);  // the following evaluation gathers v*_j of ghosts (and the velocity fold reads vel = v* for ghosts)
}

// ---- ParticlesContacts materialisation + the context-style host plugin call (nonpressure_force.rs:15-27) ---------------
struct HostContacts {
    std::vector<uint32_t> offsets, j, model;
    std::vector<float> weight, gradient;
};
// which = 0: fluid-fluid contacts, 1: fluid-boundary contacts of fluid `f`'s particles, CSR in the fluid's original order
sph_status materialise_contacts(sph_world* w, uint32_t f, int which, HostContacts* out) {
    const FluidRec& fl = w->fluids[f];
    const size_t N = w->N, Nf = fl.n;
    const int c = w->cur, bc = w->bcur;
    const uint32_t ob = w->own_begin;
    const uint32_t cap = which ? w->lists.cap_b : w->lists.cap_f;
    const uint32_t* cnt = which ? w->lists.cnt_b.p : w->lists.cnt_f.p;
    CU(w->ct_cnt[which].ensure(N + 1));
    LAUNCH(k_contacts_count, N, 256, (uint32_t)N, w->orig[c].p + ob, cnt + ob, cap, w->ct_cnt[which].p);
    CU(cudaMemsetAsync(w->ct_cnt[which].p + N, 0, sizeof(uint32_t), w->st));
    TRY(scan_exclusive(w, w->ct_cnt[which].p, N + 1));
    std::vector<uint32_t> scan(Nf + 1);
    CU(cudaMemcpyAsync(scan.data(), w->ct_cnt[which].p + fl.offset, (Nf + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
    uint32_t total = 0;
    CU(cudaMemcpyAsync(&total, w->ct_cnt[which].p + N, sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
    CU(cudaStreamSynchronize(w->st));
    CU(w->ct_j[which].ensure(std::max<size_t>(total, 1)));
    CU(w->ct_model[which].ensure(std::max<size_t>(total, 1)));
    CU(w->ct_w[which].ensure(std::max<size_t>(total, 1)));
    CU(w->ct_g[which].ensure(3 * std::max<size_t>(total, 1)));
    OffsetTable tab;
    memset(&tab, 0, sizeof tab);
    if (which) {
        for (size_t b = 0; b < w->bounds.size(); ++b) tab.off[b] = (uint32_t)w->bounds[b].offset;
        if (w->B)
            LAUNCH((k_contacts_fill<true>), N, 128, (uint32_t)N, w->pos[c].p, w->bpos[bc].p, w->bvel[bc].p, w->orig[c].p, w->borig[bc].p, w->lists.view(),
                   w->ct_cnt[which].p, tab, w->ct_j[which].p, w->ct_model[which].p, w->ct_w[which].p, w->ct_g[which].p);
    } else {
        for (size_t k = 0; k < w->fluids.size(); ++k) tab.off[k] = (uint32_t)w->fluids[k].offset;
        LAUNCH((k_contacts_fill<false>), N, 128, (uint32_t)N, w->pos[c].p, w->pos[c].p, w->vel[c].p, w->orig[c].p, w->orig[c].p, w->lists.view(),
               w->ct_cnt[which].p, tab, w->ct_j[which].p, w->ct_model[which].p, w->ct_w[which].p, w->ct_g[which].p);
    }
    const uint32_t first = scan[0], nent = scan[Nf] - scan[0];
    out->offsets.resize(Nf + 1);
    for (size_t i = 0; i <= Nf; ++i) out->offsets[i] = scan[i] - first;
    out->j.resize(nent);
    out->model.resize(nent);
    out->weight.resize(nent);
    out->gradient.resize(3 * (size_t)nent);
    if (nent) {
        CU(cudaMemcpyAsync(out->j.data(), w->ct_j[which].p + first, nent * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
        CU(cudaMemcpyAsync(out->model.data(), w->ct_model[which].p + first, nent * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
        CU(cudaMemcpyAsync(out->weight.data(), w->ct_w[which].p + first, nent * sizeof(float), cudaMemcpyDeviceToHost, w->st));
        CU(cudaMemcpyAsync(out->gradient.data(), w->ct_g[which].p + 3 * (size_t)first, 3 * (size_t)nent * sizeof(float), cudaMemcpyDeviceToHost, w->st));
    }
    CU(cudaStreamSynchronize(w->st));
    return SPH_OK;
}

sph_status call_host_force2(sph_world* w, uint32_t f, ForceRec& fr, std::vector<float>& hp, std::vector<float>& hv, std::vector<float>& hd,
                            std::vector<float>& ha) {
    if (w->slab.active && (fr.host_flags & SPH_HOST_FORCE_CONTACTS))
        return w->fail(SPH_ERR_INVALID, "materialised contacts are not available in slab-decomposed worlds");
    const FluidRec& fl = w->fluids[f];
    sph_host_force_ctx ctx;
    memset(&ctx, 0, sizeof ctx);
    ctx.dt = w->dt;
    ctx.inv_dt = w->inv_dt;
    ctx.kernel_radius = w->h;
    ctx.particle_radius = w->desc.particle_radius;
    ctx.fluid = make_handle(f, fl.gen);
    ctx.fluid_index = f;
    ctx.density0 = fl.density0;
    ctx.n = fl.n;
    ctx.positions_xyz = hp.data();
    ctx.velocities_xyz = hv.data();
    ctx.densities = hd.data();
    ctx.accelerations_xyz = ha.data();
    if (!w->slab.active) ctx.volumes = w->rows.vol.data() + fl.offset;  // a slab step does not size the host rows
    HostContacts ff, fb;
    if (fr.host_flags & SPH_HOST_FORCE_CONTACTS) {
        TRY(materialise_contacts(w, f, 0, &ff));
        TRY(materialise_contacts(w, f, 1, &fb));
        ctx.ff_offsets = ff.offsets.data(); ctx.ff_j = ff.j.data(); ctx.ff_j_model = ff.model.data();
        ctx.ff_weight = ff.weight.data(); ctx.ff_gradient_xyz = ff.gradient.data();
        ctx.fb_offsets = fb.offsets.data(); ctx.fb_j = fb.j.data(); ctx.fb_j_model = fb.model.data();
        ctx.fb_weight = fb.weight.data(); ctx.fb_gradient_xyz = fb.gradient.data();
    }
    std::vector<sph_boundary_view> views;
    std::vector<float> bvol;
    if (fr.host_flags & SPH_HOST_FORCE_BOUNDARIES) {
        bvol.resize(w->B);
        if (w->B) TRY(export_rows(w, boundary_col(w, W4{w->bpos[w->bcur].p}, 0, w->B, bvol.data())));
        TRY(pull_boundaries(w));
        views.resize(w->bounds.size());
        for (size_t b = 0; b < w->bounds.size(); ++b) {
            const BoundaryRec& br = w->bounds[b];
            views[b].n = br.alive ? br.n : 0;
            views[b].positions_xyz = w->brows.pos.data() + 3 * br.offset;
            views[b].velocities_xyz = w->brows.vel.data() + 3 * br.offset;
            views[b].volumes = bvol.data() + br.offset;
        }
        ctx.n_boundaries = views.size();
        ctx.boundaries = views.data();
    }
    fr.host_fn2(fr.host_user, &ctx);
    return SPH_OK;
}

// predict_advection dfsph_solver.rs:580-603: every fluid's forces in push order, less what the divergence loop computed
// (fold: fold_state)
sph_status phase_forces(sph_world* w, uint32_t fold) {
    size_t N = w->N;
    int c = w->cur, bc = w->bcur;
    const bool multi = w->fluids.size() > 1, bf = any_bforce(w);
    const Lists L = w->lists.view();
    for (size_t f = 0; f < w->fluids.size(); ++f)
        for (ForceRec& fr : w->fluids[f].forces) {
            const float* p = fr.d.p;
            switch (fr.d.kind) {
                case SPH_FORCE_XSPH_VISCOSITY:
                    if ((fold & FOLD_XS) && f == 0 && &fr == &w->fluids[0].forces[0]) break;  // already folded in by k_fold_velocities
                    DISPATCH2(k_force_xsph, multi, bf, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, w->bvel[bc].p, L, w->dens.p, w->acc.p,
                              w->bforce.p, (uint32_t)f, p[0], p[1], w->inv_dt);
                    break;
                case SPH_FORCE_ARTIFICIAL_VISCOSITY:
                    DISPATCH2(k_force_artificial, multi, bf, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, w->bvel[bc].p, L, w->dens.p, w->acc.p,
                              w->bforce.p, (uint32_t)f, p[0], p[1], p[2], p[3], p[4]);
                    break;
                case SPH_FORCE_AKINCI2013_TENSION: {
                    if ((fold & FOLD_AKINCI) && &fr == &w->fluids[0].forces[0]) break;  // in xs, folded in by the fold pass
                    CU(w->normals.ensure(std::max(w->Ntot, w->N)));
                    const AkinciNorms an = akinci_norms(w->h);
                    const float coh_norm = an.coh_norm, h6_64 = an.h6_64, adh_norm = an.adh_norm;
                    if ((fold & FOLD_NR4) && f == 0) {  // normals (and rho, in .w) came with the first divergence update
                        CU(w->tex_pvx.bind(w->pvx4));
                        if (bf) LAUNCH((k_akinci_force_u<true>), N, PASS_T, w->pvx4.p, w->tex_pvx.obj, w->normals.p, w->bpos[bc].p, L, w->acc.p, w->bforce.p, p[0], p[1], coh_norm, h6_64, adh_norm);
                        else LAUNCH((k_akinci_force_u<false>), N, PASS_T, w->pvx4.p, w->tex_pvx.obj, w->normals.p, w->bpos[bc].p, L, w->acc.p, w->bforce.p, p[0], p[1], coh_norm, h6_64, adh_norm);
                        break;
                    }
                    DISPATCH1(k_akinci_normals, multi, N, PASS_T, w->pos[c].p, w->vel[c].p, L, w->dens.p, w->normals.p, (uint32_t)f);
                    TRY(slab_refresh(w, w->normals.p, sizeof(float4)));
                    DISPATCH2(k_akinci_force, multi, bf, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, L, w->dens.p, w->normals.p, w->acc.p,
                              w->bforce.p, (uint32_t)f, p[0], p[1], coh_norm, h6_64, adh_norm);
                    break;
                }
                case SPH_FORCE_BECKER2009_ELASTICITY:
                    TRY(elasticity_solve(w, (uint32_t)f, fr));
                    break;
                case SPH_FORCE_HE2014_TENSION: {
                    CU(w->he_colors.ensure(std::max(w->Ntot, w->N)));
                    CU(w->he_gradc.ensure(std::max(w->Ntot, w->N)));
                    DISPATCH1(k_he2014_colors, multi, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, L, w->dens.p, w->he_colors.p, (uint32_t)f);
                    TRY(slab_refresh(w, w->he_colors.p, sizeof(float)));
                    DISPATCH1(k_he2014_gradc, multi, N, PASS_T, w->pos[c].p, w->vel[c].p, L, w->dens.p, w->he_colors.p, w->he_gradc.p, (uint32_t)f);
                    TRY(slab_refresh(w, w->he_gradc.p, sizeof(float)));
                    DISPATCH2(k_he2014_force, multi, bf, N, PASS_T, w->pos[c].p, w->vel[c].p, w->bpos[bc].p, L, w->dens.p, w->he_gradc.p, w->acc.p,
                              w->bforce.p, (uint32_t)f, p[0], p[1]);
                    break;
                }
                case SPH_FORCE_DFSPH_VISCOSITY:
                    TRY(viscosity_solve(w, (uint32_t)f, fr));
                    break;
                case SPH_FORCE_WCSPH_TENSION:
                    if (p[0] != 0.f) DISPATCH1(k_wcsph_force, multi, N, PASS_T, w->pos[c].p, w->vel[c].p, L, w->acc.p, (uint32_t)f, p[0]);
                    break;
                case FORCE_HOST_CALLBACK: {  // user-defined NonPressureForce::solve on the host (nonpressure_force.rs:10-30)
                    // called for an empty fluid too (n = 0, offsets {0}), as predict_advection calls solve for every fluid
                    FluidRec& fl = w->fluids[f];
                    const size_t Nf = fl.n;
                    std::vector<float> hp(3 * Nf), hv(3 * Nf), ha(3 * Nf), hd(Nf);
                    TRY(export_rows(w, fluid_col(w, Xyz{w->pos[c].p}, fl.offset, Nf, hp.data()), fluid_col(w, Xyz{w->vel[c].p}, fl.offset, Nf, hv.data()),
                                    fluid_col(w, Xyz{w->acc.p}, fl.offset, Nf, ha.data()), fluid_col(w, Rows<1>{w->dens.p}, fl.offset, Nf, hd.data())));
                    w->in_host_force = true;
                    sph_status hs = SPH_OK;
                    if (fr.host_fn2) hs = call_host_force2(w, (uint32_t)f, fr, hp, hv, hd, ha);
                    else fr.host_fn(fr.host_user, w->dt, w->inv_dt, w->h, Nf, hp.data(), hv.data(), hd.data(), ha.data());
                    w->in_host_force = false;
                    TRY(hs);
                    TRY(enter(w));  // the callback may have used another world of this process
                    ImportRows back;
                    back.vc = ha.data();
                    TRY(import_rows(w, back, fl.offset, Nf, w->acc.p));
                    break;
                }
                default:
                    return w->fail(SPH_ERR_INVALID, "unknown force kind %d", fr.d.kind);
            }
            fr.solved = true;
        }
    CU(cudaGetLastError());
    return SPH_OK;
}

// The CFL rule's substep count (DESIGN.md section 12): d = (r * 2) / sqrt(m) * cfl in the order of max_substep
// (timestep_manager.rs:36-46), +inf for m == 0, and n = clamp(ceil(R / d), max(1, min - k), max(1, max - k)); a non-finite
// or NaN ratio takes the upper bound
uint32_t cfl_substeps(float m, float remaining, float r, float cfl, uint32_t min_substeps, uint32_t max_substeps, uint32_t k) {
    const float d = m == 0.f ? INFINITY : r * 2.0f / sqrtf(m) * cfl;
    const int64_t lo = std::max<int64_t>(1, (int64_t)min_substeps - k), hi = std::max<int64_t>(1, (int64_t)max_substeps - k);
    const float q = ceilf(remaining / d);
    if (!(q <= (float)hi)) return (uint32_t)hi;
    return (uint32_t)std::max<int64_t>(lo, (int64_t)q);
}

// Substepping only: the CFL reduction over the velocities `vel` and this substep's accelerations, enqueued after the forces
sph_status launch_cfl_max(sph_world* w, const float4* vel, float remaining) {
    if (w->cfl_coeff == 0.f) return SPH_OK;
    CU(cudaMemsetAsync(&w->d_ss.p->cfl_bits, 0, sizeof(uint32_t), w->st));
    LAUNCH(k_cfl_max, w->N, 256, vel, w->acc.p, remaining, &w->d_ss.p->cfl_bits);
    return SPH_OK;
}

// TimestepManager::advance timestep_manager.rs:76-88: the substep is the whole remaining time R_k, or with substepping on
// R_k / n_k of the CFL rule, which reads back launch_cfl_max's result (the substep's one host synchronisation for it)
sph_status timestep_advance(sph_world* w, float remaining) {
    float dt = remaining;
    if (w->cfl_coeff != 0.f) {
        TRY(read_scalars(w, SS_BEGIN(cfl_bits), SS_END(cfl_bits)));
        CU(cudaStreamSynchronize(w->st));
        const uint32_t n = cfl_substeps(__uint_as_float_host(w->h_ss->cfl_bits), remaining, w->desc.particle_radius, w->cfl_coeff, w->min_substeps,
                                        w->max_substeps, (uint32_t)w->substeps.size());
        dt = remaining / (float)n;
    }
    w->dt = dt;
    w->inv_dt = dt == 0.f ? 0.f : 1.0f / dt;
    if (!w->cap) w->substeps.push_back(dt);
    return SPH_OK;
}

// update_velocities :422-430, zero vc :689-691, acc += gravity :574-578, the non-pressure forces and the integration, after the
// divergence loop ended in fold state `fold` (fold_state)
sph_status dfsph_fold(sph_world* w, float remaining, const float g[3], uint32_t fold) {
    size_t N = w->N;
    int c = w->cur;
    // the first force of fluid 0 may already sit in xs: the XSPH sums of the loop's last evaluation (acc = g + xs * inv_dt) or
    // the Akinci fluid force (acc = g + xs; a scale of 1 leaves the product exact)
    const bool folded = fold & (FOLD_XS | FOLD_AKINCI);
    const float4* xs = folded ? w->xs.p : nullptr;
    const float xs_scale = (fold & FOLD_AKINCI) ? 1.0f : w->inv_dt;
    // nothing (else) to launch in the force phase?  Then fold, acceleration and integration are one streaming pass, unless
    // substepping needs the CFL reduction between the fold and the integration, which takes the new dt
    bool quiet_forces = true;
    for (size_t f = 0; f < w->fluids.size() && quiet_forces; ++f)
        for (const ForceRec& fr : w->fluids[f].forces)
            if (!(folded && f == 0 && &fr == &w->fluids[0].forces[0])) quiet_forces = false;
    if (quiet_forces && w->cfl_coeff == 0.f) {
        TRY(ev_record(w, EV_FOLD));
        TRY(ev_record(w, EV_FORCES));
        TRY(timestep_advance(w, remaining));  // :702
        LAUNCH(k_fold_integrate, w->Ntot, 256, w->vel[c].p, w->vc[c].p, w->vs.p, w->acc.p, g[0], g[1], g[2], xs, xs_scale, w->dt,
               w->unimass ? w->pvx4.p : nullptr, w->unimass ? w->vyz2.p : nullptr);
    } else {
        LAUNCH(k_fold_velocities, w->Ntot, 256, w->vel[c].p, w->vc[c].p, w->vs.p, w->acc.p, g[0], g[1], g[2], xs, xs_scale,  // ghosts too (vel = v*)
               w->unimass ? (const float4*)w->pvx4.p : nullptr, w->unimass ? (const float2*)w->vyz2.p : nullptr);
        TRY(ev_record(w, EV_FOLD));
        if (!quiet_forces) TRY(phase_forces(w, fold));
        TRY(ev_record(w, EV_FORCES));
        TRY(launch_cfl_max(w, w->vel[c].p, remaining));
        TRY(timestep_advance(w, remaining));  // :702
        LAUNCH(k_integrate_acc, N, 256, w->vel[c].p, w->vc[c].p, w->vs.p, w->acc.p, w->dt, w->unimass ? w->pvx4.p : nullptr,
               w->unimass ? w->vyz2.p : nullptr);
    }
    TRY(refresh_vstar(w));
    return ev_record(w, EV_INTEG);
}

// A condition of dfsph_step's loops: out of capture a host bool that decide() sets, in capture a conditional handle
struct Cond {
    bool v = false;
    cudaGraphConditionalHandle h = 0;
};
template <class Fn>
sph_status cap_cond(sph_world* w, cudaGraphConditionalHandle h, cudaGraphConditionalNodeType type, Fn body);  // sph_graph.inl
sph_status new_handle(sph_world* w, cudaGraphConditionalHandle* h);

sph_status cond_new(sph_world* w, Cond* c) { return w->cap ? new_handle(w, &c->h) : SPH_OK; }

// IF (cudaGraphCondTypeIf) or WHILE c { body }: plain control flow out of capture, a conditional node in capture
template <class Fn>
sph_status cond(sph_world* w, const Cond& c, cudaGraphConditionalNodeType type, Fn body) {
    if (w->cap) return cap_cond(w, c.h, type, body);
    if (type == cudaGraphCondTypeIf) return c.v ? body() : SPH_OK;
    while (c.v) TRY(body());
    return SPH_OK;
}

// The decision after evaluation i of loop r (i < 0: the evaluation after the last decided one), from nblk error partials.
// It sets c[0] to "an update follows", c[1] to "an update and another evaluation follow", c[2] to "an update follows and
// ends the loop", c[3] and c[4] to false (a graph's handles keep their values from the last step); null entries are not
// set.  Out of capture it is host_decision with the step's counts; in capture k_loop_decide, behind a k_reduce_partials of the
// evaluation's partials wherever its error is read.
sph_status decide(sph_world* w, const LoopRule& r, int i, uint32_t nblk, std::array<Cond*, 5> c) {
    if (w->cap) {
        if (i < 0 || loop_decision(r, (uint32_t)i, [] { return 0.f; }).read) {  // i < 0: the device decides whether it reads
            const int nf = (int)w->fluids.size();
            k_reduce_partials<<<nf, 256, 0, w->st>>>(w->partial.p, nblk, nf, w->d_ss.p->loop_err);
        }
        Decide d{};
        for (int k = 0; k < 5; ++k)
            if (c[k]) d.h[k] = c[k]->h;
        k_loop_decide<<<1, 1, 0, w->st>>>(w->graphs.ctl.p, w->graphs.rec.p, w->d_ss.p->loop_err, r, i, d);
        CU(cudaGetLastError());
        return SPH_OK;
    }
    sph_step_stats& S = w->stats;
    LoopDecision d;
    TRY(host_decision(w, r, (r.divergence ? S.n_divergence_eval : S.n_pressure_eval)++, nblk,
                      r.divergence ? &S.last_divergence_error : &S.last_density_error, &d));
    if (!d.brk) (r.divergence ? S.n_divergence_iter : S.n_pressure_iter)++;
    const bool v[5] = {!d.brk, d.more, !d.brk && !d.more, false, false};
    for (int k = 0; k < 5; ++k)
        if (c[k]) c[k]->v = v[k];
    return SPH_OK;
}

// DFSPHSolver::step dfsph_solver.rs:667-708 for the substep with remaining time R_k.  sph_world_step and the step graph
// (sph_graph.inl) run these same loops: out of capture their conditions are host bools, in capture conditional nodes.
sph_status dfsph_step(sph_world* w, float remaining, const float g[3]) {
    size_t N = w->N;
    int c = w->cur;
    // divergence_solve :466-503 (uses the PREVIOUS step's inv_dt; 0 on the first step), unrolled where its passes depend on
    // the iteration: evaluation 0 (the neighbour search's), update 0 (with the Akinci normals), evaluation 1 (with the XSPH
    // sums or the Akinci force), then a uniform WHILE body and the update that ends a loop running out of iterations
    w->stats.n_divergence_iter = w->stats.n_divergence_eval = 0;
    const bool akf = akinci_fusable_u(w), xsf = xsph_fusable(w);
    const LoopRule rd = loop_rule(w, true);
    uint32_t nblk = w->fused_nblk;
    auto div_update = [&](bool first) -> sph_status {
        if (!first) TRY(refresh_kappa(w));  // the update gathers kappa_j of ghosts (post_density_refresh sent evaluation 0's)
        TRY(span_begin(w, SP_DIV_UPD));
        TRY(launch_vel_update(w, false, first && akf));
        return span_end(w);
    };
    auto div_eval = [&](bool first) -> sph_status {
        TRY(span_begin(w, SP_DIV_EVAL));
        TRY(launch_vel_divergence(w, false, &nblk, first && akf));
        return span_end(w);
    };
    if (rd.maxit > 0) {  // max_divergence_iter 0: no pass at all
        Cond upd0, eval1, more, tail;
        for (Cond* x : {&upd0, &eval1, &more, &tail}) TRY(cond_new(w, x));
        TRY(decide(w, rd, 0, nblk, {&upd0, &eval1, nullptr, &more, &tail}));
        TRY(cond(w, upd0, cudaGraphCondTypeIf, [&] { return div_update(true); }));
        TRY(cond(w, eval1, cudaGraphCondTypeIf, [&] {
            TRY(div_eval(true));
            return decide(w, rd, 1, nblk, {nullptr, &more, &tail});
        }));
        TRY(cond(w, more, cudaGraphCondTypeWhile, [&] {
            TRY(div_update(false));
            TRY(div_eval(false));
            return decide(w, rd, -1, nblk, {nullptr, &more, &tail});
        }));
        TRY(cond(w, tail, cudaGraphCondTypeIf, [&] { return div_update(false); }));
    }
    TRY(ev_record(w, EV_DIV));
    // the fold in the state the loop ended in: from the host's counts, or in capture one branch per state it can end in
    if (!w->cap || !(xsf || akf) || rd.maxit == 0) {
        TRY(dfsph_fold(w, remaining, g, fold_state(xsf, akf, w->stats.n_divergence_eval, w->stats.n_divergence_iter)));
    } else {
        const uint32_t states[3] = {0u, xsf ? FOLD_XS : FOLD_NR4, FOLD_NR4 | FOLD_AKINCI};
        const int n_states = xsf ? 2 : 3;
        Decide d{};
        for (int k = 0; k < n_states; ++k) TRY(new_handle(w, &d.h[states[k]]));
        k_fold_arm<<<1, 1, 0, w->st>>>(w->graphs.ctl.p, w->graphs.rec.p, xsf, akf, d);
        for (int k = 0; k < n_states; ++k)
            TRY(cap_cond(w, d.h[states[k]], cudaGraphCondTypeIf, [&] { return dfsph_fold(w, remaining, g, states[k]); }));
    }
    // pressure_solve :432-464 (with the new inv_dt): evaluation 0, a uniform WHILE body, and the update that ends a loop
    // running out of iterations
    w->stats.n_pressure_iter = w->stats.n_pressure_eval = 0;
    const LoopRule rp = loop_rule(w, false);
    auto press_update = [&]() -> sph_status {
        TRY(refresh_kappa(w));
        TRY(span_begin(w, SP_PUPD));
        TRY(launch_vel_update(w, true));
        return span_end(w);
    };
    auto press_eval = [&]() -> sph_status {
        TRY(span_begin(w, SP_PRED));
        TRY(launch_vel_divergence(w, true, &nblk));
        return span_end(w);
    };
    if (rp.maxit > 0) {  // max_pressure_iter 0: no pressure pass at all
        Cond more, tail;
        TRY(cond_new(w, &more));
        TRY(cond_new(w, &tail));
        TRY(press_eval());
        TRY(decide(w, rp, 0, nblk, {nullptr, &more, &tail}));
        TRY(cond(w, more, cudaGraphCondTypeWhile, [&] {
            TRY(press_update());
            TRY(press_eval());
            return decide(w, rp, -1, nblk, {nullptr, &more, &tail});
        }));
        TRY(cond(w, tail, cudaGraphCondTypeIf, press_update));
    }
    TRY(ev_record(w, EV_PRESS));
    {
        CellBox* next = &w->d_ss.p->next;
        if (w->cap) k_bounds_init<<<1, 1, 0, w->st>>>(next);
        else CU(cudaMemcpyAsync(next, &CELL_BOX_EMPTY, sizeof(CellBox), cudaMemcpyHostToDevice, w->st));
        LAUNCH(k_update_positions, N, 256, w->pos[c].p, w->vs.p, w->unimass ? (const float4*)w->pvx4.p : nullptr,
               w->unimass ? (const float2*)w->vyz2.p : nullptr, w->dt, w->slab.active ? nullptr : next);  // :411-420
        w->nb_pending = !w->slab.active;
    }
    CU(cudaGetLastError());
    return SPH_OK;
}

// Counters resume and pause across substeps (liquid_world.rs:84-148): `t` holds the substeps so far, `s` the one that just ran.
// Times and iteration / evaluation counts add up, max_neighbors is the widest of all, everything else is the last substep's.
void stats_merge(sph_step_stats& t, const sph_step_stats& s) {
    sph_step_stats m = s;
    m.step_ms = t.step_ms + s.step_ms;
    m.grid_ms = t.grid_ms + s.grid_ms;
    m.neighbors_ms = t.neighbors_ms + s.neighbors_ms;
    m.density_ms = t.density_ms + s.density_ms;
    m.divergence_ms = t.divergence_ms + s.divergence_ms;
    m.nonpressure_ms = t.nonpressure_ms + s.nonpressure_ms;
    m.pressure_ms = t.pressure_ms + s.pressure_ms;
    m.integrate_ms = t.integrate_ms + s.integrate_ms;
    m.n_divergence_iter = t.n_divergence_iter + s.n_divergence_iter;
    m.n_pressure_iter = t.n_pressure_iter + s.n_pressure_iter;
    m.n_divergence_eval = t.n_divergence_eval + s.n_divergence_eval;
    m.n_pressure_eval = t.n_pressure_eval + s.n_pressure_eval;
    m.max_neighbors = std::max(t.max_neighbors, s.max_neighbors);
    t = m;
}

// One substep of LiquidWorld::step (liquid_world.rs:84-148): colliders, grid, coupling, neighbours, the solver with the
// remaining time R_k, the substep's read-back and transmit_forces.  The solver pushes dt_k to w->substeps; a substep
// without fluid particles runs no solver and pushes nothing.
sph_status world_substep(sph_world* w, float remaining, const float g[3], const sph_coupling_manager* coupling, bool colliders,
                         bool b_uploaded) {
    const size_t N = w->N, k = w->substeps.size();
    for (ColliderRec& c : w->colliders) c.impulse_pending = false;
    if (colliders) TRY(colliders_update(w, b_uploaded));
    TRY(phase_grid(w));
    w->grid_ready = true;
    w->ever_stepped = true;
    if (colliders && any_contact(w)) TRY(colliders_contact(w));
    if (coupling && coupling->update_boundaries) {
        // CouplingManager::update_boundaries runs after the FLUIDS of this substep are in the grid and before the boundaries
        // are (liquid_world.rs:86-103): queries issued by the callback see the fluid particles only.  The callback may rewrite
        // boundaries (count included) and fluid positions / velocities; the grid is then rebuilt from the edited state
        // (the reference keeps edited particles in their stale cells; re-binning them is the only deviation).
        CU(cudaStreamSynchronize(w->st));
        w->in_coupling = true;
        w->lists_valid = true;  // sentinel: a fluid write in the callback clears it
        coupling->update_boundaries(coupling->user, w, w->dt, w->inv_dt, w->h, w->desc.particle_radius);
        w->in_coupling = false;
        TRY(enter(w));
        if (w->staged) return w->fail(SPH_ERR_INVALID, "update_boundaries must not add / remove fluids or particles");
        if (w->b_dirty || !w->lists_valid) {
            TRY(upload_boundaries(w));
            w->stats.n_boundary_particles = w->B;
            TRY(phase_grid(w));
        }
        w->lists_valid = false;
    }
    CU(cudaEventRecord(w->ev[EV_GRID], w->st));
    // evaluate_kernels + compute_densities (liquid_world.rs:123-134) + compute_alphas (dfsph_solver.rs:679-684).  DFSPH:
    // computed by the neighbour search itself, together with the first divergence evaluation; otherwise enqueued
    // speculatively by the neighbour phase (EV_NBR is recorded there, between the two)
    TRY(phase_neighbors(w, [](sph_world* w) -> sph_status {
        if (w->N && w->desc.solver != SPH_SOLVER_DFSPH) TRY(launch_density_alpha(w));
        return SPH_OK;
    }));
    CU(cudaEventRecord(w->ev[EV_DENS], w->st));
    if (N) {
        if (w->desc.solver == SPH_SOLVER_DFSPH) TRY(dfsph_step(w, remaining, g));
        else TRY(iisph_step(w, remaining, g));
    }
    if (colliders && N) TRY(colliders_impulse(w));  // without fluid particles no force reaches a boundary (and dt did not advance)
    CU(cudaEventRecord(w->ev[EV_END], w->st));
    TRY(read_scalars(w, SS_BEGIN(err), SS_END(next)));
    CU(cudaStreamSynchronize(w->st));
    const StepScalars& S = *w->h_ss;
    if (w->nb_pending) w->nb = S.next;
    w->nb_valid = w->nb_pending;
    w->nb_pending = false;
    CU(cudaGetLastError());
    for (size_t i = 0; i < w->colliders.size(); ++i) {  // the step's impulse: the f32 sum of its substeps', in substep order
        ColliderRec& c = w->colliders[i];
        if (!c.impulse_pending) continue;
        if (k == 0) memcpy(c.impulse, w->h_imp + 6 * i, sizeof c.impulse);
        else
            for (int j = 0; j < 6; ++j) c.impulse[j] += w->h_imp[6 * i + j];
    }
    if (!w->b_reused) w->bb_contacts = S.contacts_bb;
    w->stats.n_contacts = w->bb_contacts + S.contacts_f;
    auto el = [&](int a, int b) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, w->ev[a], w->ev[b]);
        return ms;
    };
    w->stats.step_ms = el(EV_START, EV_END);
    w->stats.grid_ms = el(EV_START, EV_GRID);
    w->stats.neighbors_ms = el(EV_GRID, EV_NBR);
    w->stats.density_ms = el(EV_NBR, EV_DENS);
    if (N && w->desc.solver == SPH_SOLVER_DFSPH) {
        w->stats.divergence_ms = el(EV_DENS, EV_DIV);
        w->stats.nonpressure_ms = el(EV_FOLD, EV_FORCES);
        w->stats.pressure_ms = el(EV_INTEG, EV_PRESS);
        w->stats.integrate_ms = el(EV_DIV, EV_FOLD) + el(EV_FORCES, EV_INTEG) + el(EV_PRESS, EV_END);
    } else if (N) {
        w->stats.nonpressure_ms = el(EV_DENS, EV_FORCES);
        w->stats.pressure_ms = el(EV_INTEG, EV_PRESS);
        w->stats.integrate_ms = el(EV_FORCES, EV_INTEG) + el(EV_PRESS, EV_END);
    }
    if (S.err & ERR_PEER_TIMEOUT) return w->fail(SPH_ERR_NCCL, "peer-memory ghost exchange timed out (a neighbour rank never delivered its boundary column)");
    if (S.err) return w->fail(SPH_ERR_ZERO_DENSITY, "zero density (reference asserts dfsph_solver.rs:92,145,662)");
    if (coupling && coupling->transmit_forces) coupling->transmit_forces(coupling->user, w, w->dt, w->inv_dt);  // liquid_world.rs:146
    return SPH_OK;
}

// LiquidWorld::step liquid_world.rs:62-158: the refusals, the pending deletes (:79-81) and the staging run once, then substeps
// until the remaining time is used up (:84, is_done timestep_manager.rs:56-58)
sph_status world_step(sph_world* w, float dt, const float g[3], const sph_coupling_manager* coupling = nullptr) {
    TRY(enter(w));
    w->launches = 0;
    w->stats_exchanges = 0;
    w->n_spans = 0;
    w->nb_pending = false;
    memset(&w->stats, 0, sizeof w->stats);
    w->substeps.clear();
    const bool colliders = any_collider(w);  // refused before anything of the step is applied
    if (colliders && coupling) return w->fail(SPH_ERR_INVALID, "registered colliders and a host coupling manager cannot run in one step");
    if (colliders && w->slab.active) return w->fail(SPH_ERR_INVALID, "colliders are not supported in slab-decomposed worlds");
    uint64_t next_ids[MAX_FLUIDS];
    TRY(edits_before_marks(w, next_ids));
    TRY(apply_pending_deletes(w));  // liquid_world.rs:79-81
    TRY(stage_up(w));
    TRY(apply_sources_sinks(w, next_ids));  // DESIGN.md section 14
    for (ColliderRec& c : w->colliders) memset(c.impulse, 0, sizeof c.impulse);
    const bool b_uploaded = w->b_dirty;
    TRY(upload_boundaries(w));
    w->stats.n_fluid_particles = w->N;
    w->stats.n_boundary_particles = w->B;
    if (w->fluids.size() > (size_t)MAX_FLUIDS || w->bounds.size() > (size_t)MAX_BOUNDARIES)
        return w->fail(SPH_ERR_INVALID, "too many fluids (max %d) or boundaries (max %d)", MAX_FLUIDS, MAX_BOUNDARIES);
    if (!(dt > F32_EPS)) return SPH_OK;  // timestep_manager.rs:56-58: is_done() before the first substep
    CU(cudaEventRecord(w->ev[EV_START], w->st));
    if (w->slab.active) {  // one substep: sph_world_set_substepping refuses slab worlds
        TRY(slab_begin_step(w));
        w->stats.n_fluid_particles = w->N;
    } else {
        w->Ntot = w->N;
        w->own_begin = 0;
    }
    if (w->Ntot + w->B == 0) return SPH_OK;
    const sph_step_stats start = w->stats;
    sph_step_stats total = start;
    sph_status s = SPH_OK;
    for (float remaining = dt;;) {
        const size_t k = w->substeps.size();
        if (k) {
            w->stats = start;
            w->stats.n_boundary_particles = w->B;
            CU(cudaEventRecord(w->ev[EV_START], w->st));
        }
        s = world_substep(w, remaining, g, coupling, colliders, b_uploaded && k == 0);
        if (k == 0) total = w->stats;
        else stats_merge(total, w->stats);
        if (s != SPH_OK || w->substeps.size() == k) break;  // failed, or no solver ran: dt did not advance
        remaining -= w->dt;                                 // R_{k+1} = R_k - dt_k
        if (!(remaining > F32_EPS)) break;
    }
    w->stats = total;
    w->stats.n_substeps = (uint32_t)w->substeps.size();
    w->stats.kernel_launches = w->launches;
    w->stats.n_ghost_particles = (uint32_t)(w->Ntot - w->N);
    w->stats.n_migrated = w->slab.migrated_in + w->slab.migrated_out;
    w->stats.n_exchanges = (uint32_t)w->stats_exchanges;
    float acc[SP_COUNT] = {0.f, 0.f, 0.f, 0.f};
    for (size_t i = 0; i < w->n_spans; ++i) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, w->spans[i].a, w->spans[i].b);
        acc[w->spans[i].slot] += ms;
    }
    w->stats.divergence_eval_ms = acc[SP_DIV_EVAL];
    w->stats.divergence_update_ms = acc[SP_DIV_UPD];
    w->stats.predict_density_ms = acc[SP_PRED];
    w->stats.pressure_update_ms = acc[SP_PUPD];
    return s;
}

}  // namespace

#include "sph_slab.inl"
#include "sph_iisph_host.inl"
#include "sph_elasticity_host.inl"
#include "sph_viscosity_host.inl"
#include "sph_colliders_host.inl"
#include "sph_graph.inl"
#include "sph_edits_host.inl"
#include "sph_surface_host.inl"
#include "sph_diffuse_host.inl"

// ===================================================================================================
// extern "C" boundary
// ===================================================================================================
extern "C" {

void sph_world_desc_default(sph_world_desc* d) {
    memset(d, 0, sizeof *d);
    d->solver = SPH_SOLVER_DFSPH;
    d->particle_radius = 0.05f;
    d->smoothing_factor = 2.0f;
    d->min_pressure_iter = 1;
    d->max_pressure_iter = 50;
    d->max_density_error = 0.05f;
    d->min_divergence_iter = 1;
    d->max_divergence_iter = 50;
    d->max_divergence_error = 0.1f;
    d->omega = 0.5f;
    d->device = 0;
    d->slab_rank = 0;
    d->slab_count = 1;
    d->deterministic = 1;
    d->gather_backend = 0;
}

sph_status sph_world_create(const sph_world_desc* desc, sph_world** out) {
    if (!desc || !out) return SPH_ERR_INVALID;
    *out = nullptr;
    if (!(desc->particle_radius > 0.f) || !(desc->smoothing_factor > 0.f)) return SPH_ERR_INVALID;
    if (desc->solver != SPH_SOLVER_DFSPH && desc->solver != SPH_SOLVER_IISPH) return SPH_ERR_INVALID;
    if (desc->kernel_density < 0 || desc->kernel_density > SPH_KERNEL_VISCOSITY || desc->kernel_gradient < 0 || desc->kernel_gradient > SPH_KERNEL_VISCOSITY)
        return SPH_ERR_INVALID;
    if (desc->gather_backend != 0) return SPH_ERR_INVALID;  // see sph_world_desc::gather_backend
#if !SPH_GENERIC_KERNELS
    // this build monomorphises the solver on CubicSplineKernel; libsalva_b200_kernels.so carries the other kernels
    if (desc->kernel_density != SPH_KERNEL_CUBIC_SPLINE || desc->kernel_gradient != SPH_KERNEL_CUBIC_SPLINE) return SPH_ERR_INVALID;
#endif
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || desc->device < 0 || desc->device >= ndev) return SPH_ERR_CUDA;
    if (cudaSetDevice(desc->device) != cudaSuccess) return SPH_ERR_CUDA;
    sph_world* w = new sph_world();
    w->desc = *desc;
    w->h = desc->particle_radius * desc->smoothing_factor * 2.0f;  // liquid_world.rs:44
    w->rows.vol0 = default_volume(desc->particle_radius);
    if (const char* t = getenv("SALVA_B200_XYSUB")) w->xysub = std::min(4, std::max(1, atoi(t)));
    memset(&w->hc, 0, sizeof w->hc);
    memset(&w->stats, 0, sizeof w->stats);
    bool ok = cudaStreamCreateWithFlags(&w->st, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < EV_COUNT; ++i) ok = cudaEventCreate(&w->ev[i]) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&w->ev_lists, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaMallocHost(&w->h_ss, sizeof(StepScalars)) == cudaSuccess;
    ok = ok && w->d_ss.ensure(1) == cudaSuccess;
    if (!ok) {
        delete w;
        return SPH_ERR_CUDA;
    }
    fill_static_consts(w);
    *out = w;
    return SPH_OK;
}

void sph_world_destroy(sph_world* w) {
    if (!w) return;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    cudaSetDevice(w->desc.device);
    if (w->st) cudaStreamSynchronize(w->st);
    slab_release(w);
    if (g_const_owner == w) g_const_owner = nullptr;
    delete w;
}

// The id rule (DESIGN.md §3) for n new particles: sph_fluid_add and sph_fluid_replace_particles without ids number a fluid
// 0..n-1 (append_to = null).  sph_fluid_append numbers upwards from 1 + the largest id of the fluid's particles, marked ones
// included: the count would repeat the id of a survivor once a delete has shrunk the fluid, and the in-cell order (fluid, id)
// needs ids to be unique.  Ids past 2^32 - 1 are refused.
static sph_status new_ids(sph_world* w, const FluidRec* append_to, size_t n, std::vector<uint32_t>* ids) {
    uint64_t next = 0;
    if (append_to)
        for (size_t i = 0; i < append_to->n; ++i) next = std::max<uint64_t>(next, (uint64_t)w->rows.gid[append_to->offset + i] + 1u);
    if (next + n > (uint64_t)UINT32_MAX + 1u)
        return w->fail(SPH_ERR_INVALID, "ids %llu.. of %zu new particles do not fit 32 bits (renumber with sph_fluid_set_ids)", (unsigned long long)next, n);
    ids->resize(n);
    for (size_t i = 0; i < n; ++i) (*ids)[i] = (uint32_t)(next + i);
    return SPH_OK;
}

sph_status sph_fluid_add(sph_world* w, const float* pos, const float* vel, const float* volumes, size_t n, float density0, uint32_t memberships,
                         uint32_t filter, uint32_t* handle) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (n && !pos) return w->fail(SPH_ERR_INVALID, "sph_fluid_add: null positions");
    size_t slot = w->fluids.size();
    for (size_t k = 0; k < w->fluids.size(); ++k)
        if (!w->fluids[k].alive) { slot = k; break; }
    if (slot >= (size_t)MAX_FLUIDS) return w->fail(SPH_ERR_INVALID, "too many fluids (max %d)", MAX_FLUIDS);
    TRY(enter(w));
    TRY(stage_down(w));
    std::vector<uint32_t> ids;
    TRY(new_ids(w, nullptr, n, &ids));
    FluidRec f;
    if (slot < w->fluids.size()) f.gen = w->fluids[slot].gen + 1;
    f.n = n;
    f.density0 = density0;
    f.memberships = memberships;
    f.filter = filter;
    f.pending_delete.assign(n, 0);
    // the host rows are ordered by slot: a reused slot's (empty) range sits at its offset
    if (slot == w->fluids.size()) w->fluids.push_back(FluidRec());
    w->fluids[slot].n = 0;
    recompute_offsets(w);
    w->rows.splice(w->fluids[slot].offset, 0, n, pos, vel, nullptr, volumes, ids.data());
    w->fluids[slot] = std::move(f);
    recompute_offsets(w);
    if (handle) *handle = make_handle(slot, w->fluids[slot].gen);
    return SPH_OK;
}

sph_status sph_fluid_push_force(sph_world* w, uint32_t fluid_h, const sph_force_desc* force) {
    if (!w || !force) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    if (force->kind < 0 || force->kind > SPH_FORCE_DFSPH_VISCOSITY) return w->fail(SPH_ERR_INVALID, "unknown force kind %d", force->kind);
    if (force->kind == SPH_FORCE_WCSPH_TENSION && force->p[1] != 0.f)
        return w->fail(SPH_ERR_INVALID,
                       "WCSPHSurfaceTension: boundary coefficient must be 0 (the reference's boundary loop indexes boundaries with fluid "
                       "contacts, wcsph_surface_tension.rs:66-83)");
    if (force->kind == SPH_FORCE_DFSPH_VISCOSITY && !(force->p[0] >= 0.f && force->p[0] <= 1.f))
        return w->fail(SPH_ERR_INVALID, "The viscosity coefficient must be between 0.0 and 1.0. (dfsph_viscosity.rs:106-110)");
    ForceRec fr;
    fr.d = *force;
    w->fluids[fluid].forces.push_back(std::move(fr));
    return SPH_OK;
}

sph_status sph_fluid_push_host_force(sph_world* w, uint32_t fluid_h, sph_host_force_fn fn, void* user) {
    if (!w || !fn) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    ForceRec fr;
    memset(&fr.d, 0, sizeof fr.d);
    fr.d.kind = FORCE_HOST_CALLBACK;
    fr.host_fn = fn;
    fr.host_user = user;
    w->fluids[fluid].forces.push_back(std::move(fr));
    return SPH_OK;
}

// Fluid::add_particles fluid.rs:126-150 — appended at the end of the fluid's index range.
sph_status sph_fluid_append(sph_world* w, uint32_t fluid_h, const float* pos, const float* vel, size_t n) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    if (n == 0) return SPH_OK;
    if (!pos) return w->fail(SPH_ERR_INVALID, "sph_fluid_append: null positions");
    TRY(enter(w));
    TRY(stage_down(w));
    FluidRec& f = w->fluids[fluid];
    std::vector<uint32_t> ids;
    TRY(new_ids(w, &f, n, &ids));
    w->rows.splice(f.offset + f.n, 0, n, pos, vel, nullptr, nullptr, ids.data());
    f.n += n;
    f.pending_delete.resize(f.n, 0);
    recompute_offsets(w);
    return SPH_OK;
}

sph_status sph_fluid_delete(sph_world* w, uint32_t fluid_h, const uint8_t* mask, size_t n) {
    if (!w || !mask) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    FluidRec& f = w->fluids[fluid];
    if (n != f.n) return w->fail(SPH_ERR_INVALID, "sph_fluid_delete: mask length %zu != particle count %zu", n, f.n);
    for (size_t i = 0; i < n; ++i)
        if (mask[i] && !f.pending_delete[i]) {
            f.pending_delete[i] = 1;
            f.n_pending++;
        }
    return SPH_OK;
}

sph_status sph_fluid_count(sph_world* w, uint32_t fluid_h, size_t* n) {
    if (!w || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    *n = w->fluids[fluid].n;
    return SPH_OK;
}

sph_status sph_fluid_write(sph_world* w, uint32_t fluid_h, const float* pos, const float* vel, size_t n) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    FluidRec& f = w->fluids[fluid];
    if (n != f.n) return w->fail(SPH_ERR_INVALID, "sph_fluid_write: length %zu != particle count %zu", n, f.n);
    if (n == 0 || (!pos && !vel)) return SPH_OK;
    if (w->staged) {
        if (pos) memcpy(w->rows.pos.data() + 3 * f.offset, pos, 3 * n * sizeof(float));
        if (vel) memcpy(w->rows.vel.data() + 3 * f.offset, vel, 3 * n * sizeof(float));
        return SPH_OK;
    }
    TRY(enter(w));
    TRY(import_rows(w, {pos, vel}, f.offset, n, w->vc[w->cur].p));
    w->lists_valid = false;
    if (pos) w->nb_valid = false;  // the cached bounds describe the positions the last step wrote
    return SPH_OK;
}

sph_status sph_fluid_read(sph_world* w, uint32_t fluid_h, float* pos, float* vel, size_t cap, size_t* n_out) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    FluidRec& f = w->fluids[fluid];
    if (n_out) *n_out = f.n;
    if (cap < f.n) return w->fail(SPH_ERR_INVALID, "sph_fluid_read: capacity %zu < particle count %zu", cap, f.n);
    if (f.n == 0 || (!pos && !vel)) return SPH_OK;
    if (w->staged) {
        if (pos) memcpy(pos, w->rows.pos.data() + 3 * f.offset, 3 * f.n * sizeof(float));
        if (vel) memcpy(vel, w->rows.vel.data() + 3 * f.offset, 3 * f.n * sizeof(float));
        return SPH_OK;
    }
    TRY(enter(w));
    const int c = w->cur;
    const Col<Xyz> p = fluid_col(w, Xyz{w->pos[c].p}, f.offset, f.n, pos), v = fluid_col(w, Xyz{w->vel[c].p}, f.offset, f.n, vel);
    if (pos && vel) return export_rows(w, p, v);
    return export_rows(w, pos ? p : v);
}

sph_status sph_boundary_add(sph_world* w, const float* pos, const float* vel, size_t n, uint32_t memberships, uint32_t filter, int want_forces,
                            uint32_t* handle) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (n && !pos) return w->fail(SPH_ERR_INVALID, "sph_boundary_add: null positions");
    TRY(pull_boundaries(w));
    size_t slot = w->bounds.size();
    for (size_t k = 0; k < w->bounds.size(); ++k)
        if (!w->bounds[k].alive) { slot = k; break; }
    if (slot >= (size_t)MAX_BOUNDARIES) return w->fail(SPH_ERR_INVALID, "too many boundaries (max %d)", MAX_BOUNDARIES);
    BoundaryRec b;
    if (slot < w->bounds.size()) b.gen = w->bounds[slot].gen + 1;
    b.n = n;
    b.memberships = memberships;
    b.filter = filter;
    b.want_forces = want_forces != 0;
    if (slot == w->bounds.size()) w->bounds.push_back(BoundaryRec());
    w->bounds[slot].n = 0;
    recompute_offsets(w);
    w->brows.splice(w->bounds[slot].offset, 0, n, pos, vel);
    w->bounds[slot] = b;
    recompute_offsets(w);
    w->b_dirty = true;
    if (handle) *handle = make_handle(slot, b.gen);
    return SPH_OK;
}

sph_status sph_boundary_write(sph_world* w, uint32_t boundary_h, const float* pos, const float* vel, size_t n) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    BoundaryRec& b = w->bounds[boundary];
    if (n != b.n) return w->fail(SPH_ERR_INVALID, "sph_boundary_write: length %zu != particle count %zu", n, b.n);
    if (boundary_coupled(w, boundary)) return w->fail(SPH_ERR_INVALID, "sph_boundary_write: the boundary is coupled to a collider");
    TRY(pull_boundaries(w));
    if (pos) memcpy(w->brows.pos.data() + 3 * b.offset, pos, 3 * n * sizeof(float));
    if (vel) memcpy(w->brows.vel.data() + 3 * b.offset, vel, 3 * n * sizeof(float));
    w->b_dirty = true;
    return SPH_OK;
}

static sph_status boundary_export(sph_world* w, uint32_t boundary_h, float* out, size_t cap, bool forces) {
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    BoundaryRec& b = w->bounds[boundary];
    if (cap < b.n) return w->fail(SPH_ERR_INVALID, "capacity %zu < boundary particle count %zu", cap, b.n);
    if (b.n == 0) return SPH_OK;
    size_t width = forces ? 3 : 1;
    if (w->b_dirty || (forces && !b.want_forces)) {
        memset(out, 0, width * b.n * sizeof(float));
        return SPH_OK;
    }
    TRY(enter(w));
    if (forces) return export_rows(w, boundary_col(w, Rows<3>{w->bforce.p}, b.offset, b.n, out));  // bforce: 3 floats per sorted slot
    return export_rows(w, boundary_col(w, W4{w->bpos[w->bcur].p}, b.offset, b.n, out));
}

sph_status sph_boundary_read_forces(sph_world* w, uint32_t boundary, float* f_xyz, size_t cap) {
    if (!w || !f_xyz) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return boundary_export(w, boundary, f_xyz, cap, true);
}
sph_status sph_boundary_read_volumes(sph_world* w, uint32_t boundary, float* volumes, size_t cap) {
    if (!w || !volumes) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return boundary_export(w, boundary, volumes, cap, false);
}


// LiquidWorld::particles_intersecting_aabb liquid_world.rs:211-243
sph_status sph_world_particles_in_aabb(sph_world* w, const float mins[3], const float maxs[3], uint32_t* kinds, uint32_t* handles, uint32_t* indices,
                                       size_t cap, size_t* n) {
    if (!w || !mins || !maxs || !n || (cap && (!kinds || !handles || !indices))) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    AabbQuery q;
    memset(&q, 0, sizeof q);
    q.kind = 0;
    return run_query(w, q, mins, maxs, kinds, handles, indices, cap, n);
}

// LiquidWorld::particles_intersecting_shape liquid_world.rs:246-281 for the shapes a C ABI can name: ball, cuboid, capsule
// (parry's Shape trait objects cannot cross the boundary).  The cells come from the shape's AABB under `pos`, exactly
// as `shape.compute_aabb(pos)` feeds cells_intersecting_aabb; the test is distance_to_point(pos, p, solid) <= particle_radius.
sph_status sph_world_particles_in_shape(sph_world* w, const sph_shape* shape, const float translation[3], const float rotation_rowmajor[9], uint32_t* kinds,
                                        uint32_t* handles, uint32_t* indices, size_t cap, size_t* n) {
    if (!w || !shape || !translation || !n || (cap && (!kinds || !handles || !indices))) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return particles_in_shape(w, shape, translation, rotation_rowmajor, kinds, handles, indices, cap, n);
}

// particles_intersecting_shape liquid_world.rs:246-281 for a parry HeightField: the cells of compute_aabb(pos) (centre
// R c + t), every particle in them whose distance_to_point(pos, p, solid) (is_inside is always false: the unsigned distance
// to the closest point) is <= particle_radius.  The heights live in the sampler's scratch for the call.
sph_status sph_world_particles_in_heightfield(sph_world* w, const sph_heightfield* hf, const float translation[3], const float rotation_rowmajor[9],
                                              uint32_t* kinds, uint32_t* handles, uint32_t* indices, size_t cap, size_t* n) {
    if (!w || !translation || !n || (cap && (!kinds || !handles || !indices))) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return particles_in_heightfield(w, hf, translation, rotation_rowmajor, kinds, handles, indices, cap, n);
}

// salva3d::sampling::shape_{surface,volume}_ray_sample ray_sampling.rs:9-231 (sph_sampling.cuh, DESIGN.md section 11)
sph_status sph_world_sample_shape(sph_world* w, int32_t method, const sph_shape* shape, const sph_heightfield* hf, float particle_radius,
                                  float* xyz, size_t cap, size_t* n) {
    if (!w || !shape || !n || (cap && !xyz)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return sample_shape(w, method, shape, hf, particle_radius, xyz, cap, n);
}

sph_status sph_world_step(sph_world* w, float dt, const float gravity[3]) {
    if (!w || !gravity) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "sph_world_step called from inside a coupling callback");
    sph_status s = world_step(w, dt, gravity);
    w->records.assign(1, step_record(w->stats, 0));
    if (s != SPH_OK) cudaStreamSynchronize(w->st);
    return s;
}

// n_steps calls of sph_world_step, steps 2..n_steps in a CUDA graph (DESIGN.md section 13)
sph_status sph_world_step_many(sph_world* w, float dt, const float gravity[3], uint32_t n_steps, uint32_t* steps_done) {
    if (!w || !gravity || !steps_done) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    *steps_done = 0;
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "sph_world_step_many called from inside a coupling callback");
    if (const char* why = step_many_refusal(w)) return w->fail(SPH_ERR_INVALID, "%s", why);
    if (n_steps == 0) return SPH_OK;
    sph_status s = step_many(w, dt, gravity, n_steps, steps_done);
    if (s != SPH_OK) cudaStreamSynchronize(w->st);
    return s;
}

sph_status sph_world_read_step_records(sph_world* w, sph_step_record* out, size_t cap, size_t* n) {
    if (!w || !n || (cap && !out)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    *n = w->records.size();
    if (*n && cap) memcpy(out, w->records.data(), std::min(cap, *n) * sizeof(sph_step_record));
    return SPH_OK;
}

// LiquidWorld::step_with_coupling liquid_world.rs:67-158
sph_status sph_world_step_with_coupling(sph_world* w, float dt, const float gravity[3], const sph_coupling_manager* coupling) {
    if (!w || !gravity) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "sph_world_step_with_coupling called from inside a coupling callback");
    if (coupling && w->slab.active) return w->fail(SPH_ERR_INVALID, "coupling callbacks are not supported in slab-decomposed worlds");
    sph_status s = world_step(w, dt, gravity, coupling);
    w->records.assign(1, step_record(w->stats, 0));
    w->in_coupling = false;
    if (s != SPH_OK) cudaStreamSynchronize(w->st);
    return s;
}

sph_status sph_world_force_iterations(sph_world* w, int32_t n_div, int32_t n_press) {
    if (!w) return SPH_ERR_INVALID;
    w->force_div = n_div;
    w->force_press = n_press;
    return SPH_OK;
}

// TimestepManager's cfl_coeff / min_num_substeps / max_num_substeps (timestep_manager.rs:21-46), applied with the even split of
// DESIGN.md section 12 in place of the commented-out clamp of compute_substep (:87-94)
sph_status sph_world_set_substepping(sph_world* w, float cfl_coeff, uint32_t min_substeps, uint32_t max_substeps) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (!(cfl_coeff >= 0.f)) return w->fail(SPH_ERR_INVALID, "cfl_coeff must be 0 (off) or positive, got %g", (double)cfl_coeff);
    if (min_substeps == 0 || min_substeps > max_substeps)
        return w->fail(SPH_ERR_INVALID, "substep bounds need 1 <= min_substeps <= max_substeps, got %u, %u", min_substeps, max_substeps);
    if (w->desc.slab_count > 1 || w->slab.active) return w->fail(SPH_ERR_INVALID, "substepping is not supported in slab-decomposed worlds");
    w->cfl_coeff = cfl_coeff;
    w->min_substeps = min_substeps;
    w->max_substeps = max_substeps;
    return SPH_OK;
}

sph_status sph_world_read_substeps(sph_world* w, float* dts, size_t cap, size_t* n) {
    if (!w || !n || (cap && !dts)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    *n = w->substeps.size();
    if (*n && cap) memcpy(dts, w->substeps.data(), std::min(cap, *n) * sizeof(float));
    return SPH_OK;
}

sph_status sph_world_stats(sph_world* w, sph_step_stats* out) {
    if (!w || !out) return SPH_ERR_INVALID;
    *out = w->stats;
    return SPH_OK;
}

float sph_world_h(const sph_world* w) { return w ? w->h : 0.f; }
float sph_world_particle_radius(const sph_world* w) { return w ? w->desc.particle_radius : 0.f; }

sph_status sph_debug_read(sph_world* w, uint32_t fluid_h, int what, float* out, size_t cap) {
    if (!w || !out) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    FluidRec& f = w->fluids[fluid];
    bool vec = what == SPH_DBG_VELOCITY_CHANGE || what == SPH_DBG_ACCELERATION || what == SPH_DBG_IISPH_DII || what == SPH_DBG_IISPH_DIJ_PJL;
    size_t width = vec ? 3 : 1;
    if (cap < f.n) return w->fail(SPH_ERR_INVALID, "sph_debug_read: capacity %zu < particle count %zu", cap, f.n);
    if (what >= SPH_DBG_DIFFUSE_NORMAL && what <= SPH_DBG_DIFFUSE_COUNT) return diffuse_debug_read(w, fluid, what, out);
    const bool iisph_sel = what == SPH_DBG_IISPH_DII || what == SPH_DBG_IISPH_AII || what == SPH_DBG_IISPH_DIJ_PJL;
    if (iisph_sel && (w->desc.solver != SPH_SOLVER_IISPH || !w->iisph.dii.p || w->own_begin + w->N > w->iisph.cap))
        return w->fail(SPH_ERR_INVALID, "sph_debug_read: selector %d needs an IISPH world that has stepped with its current particles", what);
    // plugin scratch: that of the fluid's last force of the selector's kind, solved since its particles last changed
    const ForceRec* pf = nullptr;
    if (what >= SPH_DBG_HE2014_COLOR && what <= SPH_DBG_EL_STRESS) {
        static const uint32_t widths[] = {1, 1, 36, 6, 1, 9, 9, 6};
        width = widths[what - SPH_DBG_HE2014_COLOR];
        const int kind = what <= SPH_DBG_HE2014_GRADC ? SPH_FORCE_HE2014_TENSION
                         : what <= SPH_DBG_VISC_TARGET ? SPH_FORCE_DFSPH_VISCOSITY : SPH_FORCE_BECKER2009_ELASTICITY;
        for (const ForceRec& fr : f.forces)
            if (fr.d.kind == kind) pf = &fr;
        const bool el = kind == SPH_FORCE_BECKER2009_ELASTICITY;
        if (!pf || w->staged || !pf->solved || (el && (!pf->elastic || pf->elastic->n != f.n)))
            return w->fail(SPH_ERR_INVALID, "sph_debug_read: selector %d needs a force of kind %d solved with the fluid's current particles", what, kind);
    }
    if (f.n == 0) return SPH_OK;
    if (w->staged) {
        // the carried state is on the host between an edit and the next step; the step's scratch reads as zero until then
        if (what == SPH_DBG_VELOCITY_CHANGE) memcpy(out, w->rows.vc.data() + 3 * f.offset, 3 * f.n * sizeof(float));
        else if (what == SPH_DBG_PRESSURE) memcpy(out, w->rows.press.data() + f.offset, f.n * sizeof(float));
        else memset(out, 0, width * f.n * sizeof(float));
        return SPH_OK;
    }
    TRY(enter(w));
    if (pf && pf->elastic) {  // the rest pose is kept in the fluid's original order already
        const ElasticityState& E = *pf->elastic;
        if (what == SPH_DBG_EL_VOLUME0) return export_rows(w, Col<W4>{{E.pos0.p}, nullptr, 0u, (uint32_t)f.n, 0, f.n, out});
        const float* src = what == SPH_DBG_EL_ROTATION ? E.rot.p : what == SPH_DBG_EL_GRAD_TR ? E.grad_tr.p : E.stress.p;
        CU(cudaMemcpyAsync(out, src, width * f.n * sizeof(float), cudaMemcpyDeviceToHost, w->st));
        CU(cudaStreamSynchronize(w->st));
        return SPH_OK;
    }
    const int c = w->cur;
    // a source that does not exist (the pressures of a DFSPH world) is refused like an unknown selector
    auto read = [&](auto src) {
        return src.p ? export_rows(w, fluid_col(w, src, f.offset, f.n, out)) : w->fail(SPH_ERR_INVALID, "sph_debug_read: unknown selector %d", what);
    };
    switch (what) {
        case SPH_DBG_DENSITY: return read(Rows<1>{w->dens.p});
        case SPH_DBG_ALPHA: return read(Rows<1>{w->alpha.p});
        case SPH_DBG_DIVERGENCE: return read(Rows<1>{w->divv.p});
        case SPH_DBG_PREDICTED_DENSITY: return read(Rows<1>{w->desc.solver == SPH_SOLVER_IISPH ? iisph_pred(w) : w->pred.p});
        case SPH_DBG_PRESSURE: return read(Rows<1>{w->press[c].p});
        case SPH_DBG_IISPH_AII: return read(Rows<1>{w->iisph.aii.p});
        case SPH_DBG_HE2014_COLOR: return read(Rows<1>{w->he_colors.p});
        case SPH_DBG_HE2014_GRADC: return read(Rows<1>{w->he_gradc.p});
        case SPH_DBG_VELOCITY_CHANGE: return read(Xyz{w->vc[c].p});
        case SPH_DBG_ACCELERATION: return read(Xyz{w->acc.p});
        case SPH_DBG_IISPH_DII: return read(Xyz{w->iisph.dii.p});
        case SPH_DBG_IISPH_DIJ_PJL: return read(Xyz{w->iisph.dij_pjl.p});
        case SPH_DBG_VISC_BETA: return read(Planes{36u, w->stride, w->visc.beta.p});
        case SPH_DBG_VISC_TARGET: return read(Planes{6u, w->stride, w->visc.target.p});
        case SPH_DBG_NUM_FLUID_CONTACTS: return read(U32<float>{w->lists.cnt_f.p});
        case SPH_DBG_NUM_BOUNDARY_CONTACTS: return read(U32<float>{w->lists.cnt_b.p});
        default: return w->fail(SPH_ERR_INVALID, "sph_debug_read: unknown selector %d", what);
    }
}

const char* sph_last_error(const sph_world* w) { return w ? w->err.c_str() : "null world"; }
const char* sph_version(void) {
#if SPH_GENERIC_KERNELS
    return "salva_b200 0.2 (sm_90a, kernels: cubic-spline poly6 spiky viscosity)";
#else
    return "salva_b200 0.2 (sm_90a, kernels: cubic-spline)";
#endif
}

sph_status sph_nccl_unique_id(char out[128]) {
    if (!out) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    std::string err;
    if (!nccl_load(&err)) return SPH_ERR_NCCL;
    nccl_uid id;
    if (g_nccl.GetUniqueId(&id) != 0) return SPH_ERR_NCCL;
    memcpy(out, id.internal, 128);
    return SPH_OK;
}

static sph_status slab_attach(sph_world* w, void* comm, bool own, int rank, int nranks) {
    if (rank < 0 || nranks < 1 || rank >= nranks) return w->fail(SPH_ERR_INVALID, "bad rank %d of %d", rank, nranks);
    SlabState& S = w->slab;
    S.comm = comm;
    S.own_comm = own;
    S.rank = rank;
    S.nranks = nranks;
    S.has_left = rank > 0;
    S.has_right = rank + 1 < nranks;
    S.active = nranks > 1;
    w->desc.deterministic = 1;  // ghost-column order agreement relies on the stable in-cell order
    CU(S.d_cnt.ensure(32));
    CU(S.d_cnt64.ensure(1));
    if (S.active) TRY(p2p_setup(w));
    return SPH_OK;
}

sph_status sph_world_attach_nccl(sph_world* w, void* nccl_comm, int rank, int nranks) {
    if (!w || !nccl_comm) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (!nccl_load(&w->err)) return SPH_ERR_NCCL;
    TRY(enter(w));
    return slab_attach(w, nccl_comm, false, rank, nranks);
}

sph_status sph_world_create_nccl(sph_world* w, const char unique_id[128], int rank, int nranks) {
    if (!w || !unique_id) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (!nccl_load(&w->err)) return SPH_ERR_NCCL;
    TRY(enter(w));
    nccl_uid id;
    memcpy(id.internal, unique_id, 128);
    void* comm = nullptr;
    NC(g_nccl.CommInitRank(&comm, nranks, id, rank));
    return slab_attach(w, comm, true, rank, nranks);
}

sph_status sph_world_set_slab(sph_world* w, int32_t cell_lo, int32_t cell_hi) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if ((long long)cell_hi - (long long)cell_lo < 2) return w->fail(SPH_ERR_INVALID, "a slab must be at least 2 cell columns wide");
    w->slab.lo = cell_lo;
    w->slab.hi = cell_hi;
    return SPH_OK;
}

sph_status sph_fluid_set_ids(sph_world* w, uint32_t fluid_h, const uint32_t* ids, size_t n) {
    if (!w || !ids) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    FluidRec& f = w->fluids[fluid];
    if (n != f.n) return w->fail(SPH_ERR_INVALID, "sph_fluid_set_ids: length %zu != particle count %zu", n, f.n);
    TRY(enter(w));
    TRY(stage_down(w));
    memcpy(w->rows.gid.data() + f.offset, ids, n * sizeof(uint32_t));
    return SPH_OK;
}

sph_status sph_fluid_read_ids(sph_world* w, uint32_t fluid_h, uint32_t* ids, size_t cap) {
    if (!w || !ids) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    FluidRec& f = w->fluids[fluid];
    if (cap < f.n) return w->fail(SPH_ERR_INVALID, "sph_fluid_read_ids: capacity %zu < particle count %zu", cap, f.n);
    if (f.n == 0) return SPH_OK;
    if (w->staged) {
        memcpy(ids, w->rows.gid.data() + f.offset, f.n * sizeof(uint32_t));
        return SPH_OK;
    }
    TRY(enter(w));
    return export_rows(w, fluid_col(w, U32<uint32_t>{w->gid[w->cur].p}, f.offset, f.n, ids));
}


// fluid.nonpressure_forces.push(Box<dyn NonPressureForce>) with the FULL solve() argument list (nonpressure_force.rs:15-27):
// timestep, kernel radius, fluid-fluid and fluid-boundary contacts, the fluid, the boundaries, the densities.
sph_status sph_fluid_push_host_force2(sph_world* w, uint32_t fluid_h, sph_host_force_fn2 fn, void* user, uint32_t flags) {
    if (!w || !fn) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    ForceRec fr;
    memset(&fr.d, 0, sizeof fr.d);
    fr.d.kind = FORCE_HOST_CALLBACK;
    fr.host_fn2 = fn;
    fr.host_flags = flags;
    fr.host_user = user;
    w->fluids[fluid].forces.push_back(std::move(fr));
    return SPH_OK;
}

// LiquidWorld::remove_fluid liquid_world.rs:171-173.  The handle dies; other handles stay valid (arena semantics).
sph_status sph_fluid_remove(sph_world* w, uint32_t fluid_h) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "fluids cannot be removed from inside a coupling callback");
    if (w->slab.active) return w->fail(SPH_ERR_INVALID, "sph_fluid_remove is not supported in slab-decomposed worlds");
    TRY(enter(w));
    TRY(stage_down(w));
    FluidRec& f = w->fluids[fluid];
    w->rows.splice(f.offset, f.n, 0, nullptr, nullptr, nullptr, nullptr, nullptr);
    f.forces.clear();
    f.pending_delete.clear();
    for (SinkRec& s : w->sinks)
        if (s.fluid == fluid) s.alive = false;
    for (SourceRec& s : w->sources)
        if (s.fluid == fluid && s.alive) {
            s.pos.release();
            s.vel.release();
            s.alive = false;
        }
    f.n_pending = 0;
    f.n = 0;
    f.alive = false;
    recompute_offsets(w);
    return SPH_OK;
}

// LiquidWorld::remove_boundary liquid_world.rs:176-178
sph_status sph_boundary_remove(sph_world* w, uint32_t boundary_h) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    TRY(pull_boundaries(w));
    BoundaryRec& b = w->bounds[boundary];
    w->brows.splice(b.offset, b.n, 0, nullptr, nullptr);
    b.n = 0;
    b.alive = false;
    b.want_forces = false;
    recompute_offsets(w);
    w->b_dirty = true;
    return SPH_OK;
}

// A coupled collider re-samples its boundary every step (positions.clear(); push(..) — fluids_pipeline.rs:175-245): the
// particle COUNT changes, which sph_boundary_write cannot express.
sph_status sph_boundary_set_particles(sph_world* w, uint32_t boundary_h, const float* pos, const float* vel, size_t n) {
    if (!w || (n && !pos)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    if (boundary_coupled(w, boundary)) return w->fail(SPH_ERR_INVALID, "sph_boundary_set_particles: the boundary is coupled to a collider");
    TRY(pull_boundaries(w));
    BoundaryRec& b = w->bounds[boundary];
    w->brows.splice(b.offset, b.n, n, pos, vel);
    b.n = n;
    recompute_offsets(w);
    w->b_dirty = true;
    return SPH_OK;
}

sph_status sph_boundary_count(sph_world* w, uint32_t boundary_h, size_t* n) {
    if (!w || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    *n = w->bounds[boundary].n;
    return SPH_OK;
}

// boundary.positions / velocities boundary.rs:13-15
sph_status sph_boundary_read(sph_world* w, uint32_t boundary_h, float* pos, float* vel, size_t cap, size_t* n) {
    if (!w || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    const BoundaryRec& b = w->bounds[boundary];
    *n = b.n;
    if ((pos || vel) && cap < b.n) return w->fail(SPH_ERR_INVALID, "sph_boundary_read: capacity %zu < particle count %zu", cap, b.n);
    TRY(pull_boundaries(w));
    if (pos) memcpy(pos, w->brows.pos.data() + 3 * b.offset, 3 * b.n * sizeof(float));
    if (vel) memcpy(vel, w->brows.vel.data() + 3 * b.offset, 3 * b.n * sizeof(float));
    return SPH_OK;
}

// The rules every registration shares: not from a callback, not in a slab world, a live boundary not coupled yet.
static sph_status collider_check_boundary(sph_world* w, uint32_t boundary_h) {
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "colliders cannot be registered from inside a coupling callback");
    if (w->slab.active) return w->fail(SPH_ERR_INVALID, "colliders are not supported in slab-decomposed worlds");
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    if (boundary_coupled(w, boundary)) return w->fail(SPH_ERR_INVALID, "boundary %u is already coupled to a collider", (unsigned)boundary_h);
    return SPH_OK;
}

// ColliderCouplingSet::register_coupling fluids_pipeline.rs:98-114
sph_status sph_collider_register(sph_world* w, uint32_t boundary_h, int32_t sampling, const sph_shape* shape, const float* pts, size_t n,
                                 uint32_t* collider) {
    if (!w || !collider || (n && !pts)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    TRY(collider_check_boundary(w, boundary_h));
    BOUNDARY_OR_FAIL(boundary, boundary_h)
    if (shape && !shape_nparams(shape->kind)) return w->fail(SPH_ERR_INVALID, "unknown shape kind %d", shape->kind);
    if (sampling != SPH_SAMPLING_STATIC && sampling != SPH_SAMPLING_CONTACT) return w->fail(SPH_ERR_INVALID, "unknown sampling %d", sampling);
    if (sampling == SPH_SAMPLING_CONTACT) {
        if (!shape) return w->fail(SPH_ERR_INVALID, "DynamicContactSampling needs the collider's shape");
        if (n) return w->fail(SPH_ERR_INVALID, "DynamicContactSampling takes no sample points");
        const int np = shape_nparams(shape->kind);
        for (int a = 0; a < np; ++a)
            if (!(std::isfinite(shape->p[a]) && shape->p[a] >= 0.f)) return w->fail(SPH_ERR_INVALID, "shape parameters must be finite and >= 0");
    }
    if (n >= (size_t)UINT32_MAX) return w->fail(SPH_ERR_INVALID, "too many sample points");
    for (size_t k = 0; k < 3 * n; ++k)
        if (!std::isfinite(pts[k])) return w->fail(SPH_ERR_INVALID, "non-finite sample point");
    size_t slot;
    TRY(collider_reserve(w, &slot));
    ColliderRec c;
    if (shape) c.shape = *shape;
    c.n = n;
    if (n) {
        std::vector<float4> l(n);
        for (size_t k = 0; k < n; ++k) l[k] = make_float4(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2], 0.f);
        CU(c.local.ensure(n));
        CU(cudaMemcpyAsync(c.local.p, l.data(), n * sizeof(float4), cudaMemcpyHostToDevice, w->st));
        CU(cudaStreamSynchronize(w->st));
    }
    // StaticSampling: the points become the boundary's particle set, and the next step poses them.  DynamicContactSampling:
    // the boundary keeps its particles until the next step samples it.
    if (sampling == SPH_SAMPLING_STATIC) {
        TRY(pull_boundaries(w));
        BoundaryRec& b = w->bounds[boundary];
        w->brows.splice(b.offset, b.n, n, pts, nullptr);
        b.n = n;
        recompute_offsets(w);
        w->b_dirty = true;
    }
    collider_commit(w, slot, boundary_h, sampling, std::move(c), collider);
    return SPH_OK;
}

// register_coupling(boundary, collider, DynamicContactSampling) for a collider whose shape is a parry HeightField: the
// heights are copied into device memory the record owns (freed by unregister and by sph_world_destroy).
sph_status sph_collider_register_heightfield(sph_world* w, uint32_t boundary_h, const sph_heightfield* hf, uint32_t* collider) {
    if (!w || !collider) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    TRY(collider_check_boundary(w, boundary_h));
    std::vector<float> heights;
    ColliderRec c;
    TRY(hf_check(w, hf, heights, c.hf, &c.hf_ylo, &c.hf_yhi));
    size_t slot;
    TRY(collider_reserve(w, &slot));
    {
        const cudaError_t e = c.hgt.ensure(heights.size());
        if (e != cudaSuccess) return w->fail(SPH_ERR_OOM, "heightfield collider: %s", cudaGetErrorString(e));
    }
    cudaError_t e = cudaMemcpyAsync(c.hgt.p, heights.data(), heights.size() * sizeof(float), cudaMemcpyHostToDevice, w->st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(w->st);
    if (e != cudaSuccess) return w->fail(SPH_ERR_CUDA, "heightfield collider upload: %s", cudaGetErrorString(e));
    c.hf.hgt = c.hgt.p;
    c.shape.kind = SPH_SHAPE_HEIGHTFIELD;
    collider_commit(w, slot, boundary_h, SPH_SAMPLING_CONTACT, std::move(c), collider);
    return SPH_OK;
}

#define COLLIDER_OR_FAIL(var, handle)                                                                   \
    const int var##_slot_ = collider_slot(w, handle);                                                   \
    if (var##_slot_ < 0) return w->fail(SPH_ERR_INVALID, "bad collider handle %u", (unsigned)(handle)); \
    ColliderRec& var = w->colliders[var##_slot_];

sph_status sph_collider_set_state(sph_world* w, uint32_t collider_h, const sph_collider_state* state) {
    if (!w || !state) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    COLLIDER_OR_FAIL(c, collider_h)
    if (state->body < SPH_BODY_NONE || state->body > SPH_BODY_DYNAMIC) return w->fail(SPH_ERR_INVALID, "unknown body kind %d", state->body);
    const float* f[5] = {state->translation, state->rotation_rowmajor, state->linvel, state->angvel, state->world_com};
    const int len[5] = {3, 9, 3, 3, 3};
    for (int a = 0; a < 5; ++a)
        for (int k = 0; k < len[a]; ++k)
            if (!std::isfinite(f[a][k])) return w->fail(SPH_ERR_INVALID, "non-finite collider state");
    c.state = *state;
    return SPH_OK;
}

// transmit_forces fluids_pipeline.rs:263-287 of the last step
sph_status sph_collider_read_impulse(sph_world* w, uint32_t collider_h, float linear[3], float angular[3]) {
    if (!w || !linear || !angular) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    COLLIDER_OR_FAIL(c, collider_h)
    const bool inert = boundary_slot(w, c.boundary) < 0;
    for (int a = 0; a < 3; ++a) {
        linear[a] = inert ? 0.f : c.impulse[a];
        angular[a] = inert ? 0.f : c.impulse[3 + a];
    }
    return SPH_OK;
}

// ColliderCouplingSet::unregister_coupling fluids_pipeline.rs:119-122
sph_status sph_collider_unregister(sph_world* w, uint32_t collider_h) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "colliders cannot be unregistered from inside a coupling callback");
    COLLIDER_OR_FAIL(c, collider_h)
    TRY(enter(w));
    c.local.release();
    c.hgt.release();
    c.alive = false;
    return SPH_OK;
}

// ---- particle sinks and sources (faucet3.rs:69-105, DESIGN.md section 14) ----------------------------------------------
// Fluid::delete_particle_at_next_timestep for every particle in (or, outside = 1, not in) a box, every step (faucet3.rs:74-86)
sph_status sph_fluid_add_sink(sph_world* w, uint32_t fluid_h, const sph_sink_desc* sink, uint32_t* handle) {
    if (!w || !sink) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    for (int a = 0; a < 3; ++a)
        if (std::isnan(sink->lo[a]) || std::isnan(sink->hi[a]) || sink->lo[a] > sink->hi[a])
            return w->fail(SPH_ERR_INVALID, "sph_fluid_add_sink: axis %d needs lo <= hi without NaN, got [%g, %g)", a, (double)sink->lo[a], (double)sink->hi[a]);
    if (sink->outside != 0 && sink->outside != 1) return w->fail(SPH_ERR_INVALID, "sph_fluid_add_sink: outside must be 0 or 1, got %d", sink->outside);
    TRY(edits_check_world(w));
    const int slot = edits_slot(w->sinks, MAX_SINKS);
    if (slot < 0) return w->fail(SPH_ERR_INVALID, "too many particle sinks (max %d)", MAX_SINKS);
    SinkRec& r = w->sinks[slot];
    r.d = *sink;
    r.fluid = fluid;
    r.alive = true;
    r.gen++;
    if (handle) *handle = make_handle(slot, r.gen & 0xFFFFu);
    return SPH_OK;
}

sph_status sph_sink_remove(sph_world* w, uint32_t sink_h) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const int slot = edits_lookup(w->sinks, sink_h);
    if (slot < 0) return w->fail(SPH_ERR_INVALID, "bad sink handle %u", (unsigned)sink_h);
    w->sinks[slot].alive = false;
    return SPH_OK;
}

// Fluid::add_particles of the same template every `interval` steps (faucet3.rs:88-103 adds a 10 x 10 sheet every 0.06 s)
sph_status sph_fluid_add_source(sph_world* w, uint32_t fluid_h, const float* pos, const float* vel, size_t n, uint32_t interval, uint32_t* handle) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    if (!pos || n == 0) return w->fail(SPH_ERR_INVALID, "sph_fluid_add_source: empty template");
    if (interval == 0) return w->fail(SPH_ERR_INVALID, "sph_fluid_add_source: interval must be at least 1 step");
    if (n > UINT32_MAX) return w->fail(SPH_ERR_INVALID, "sph_fluid_add_source: template of %zu particles is too large", n);
    TRY(edits_check_world(w));
    std::vector<float4> p(n), v(vel ? n : 0);
    CellBox cells = CELL_BOX_EMPTY;
    for (size_t i = 0; i < n; ++i) {
        p[i] = make_float4(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], 0.f);
        if (vel) v[i] = make_float4(vel[3 * i], vel[3 * i + 1], vel[3 * i + 2], 0.f);
        cell_box_add(cells, pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], w->h);
    }
    SourceRec r;
    CU(r.pos.ensure(n));
    CU(cudaMemcpy(r.pos.p, p.data(), n * sizeof(float4), cudaMemcpyHostToDevice));
    if (vel) {
        CU(r.vel.ensure(n));
        CU(cudaMemcpy(r.vel.p, v.data(), n * sizeof(float4), cudaMemcpyHostToDevice));
    }
    const int slot = edits_slot(w->sources, MAX_SOURCES);
    if (slot < 0) return w->fail(SPH_ERR_INVALID, "too many particle sources (max %d)", MAX_SOURCES);
    r.fluid = fluid;
    r.n = n;
    r.has_vel = vel != nullptr;
    r.interval = interval;
    r.age = 0;
    r.cells = cells;
    r.gen = w->sources[slot].gen + 1;
    w->sources[slot] = std::move(r);
    if (handle) *handle = make_handle(slot, w->sources[slot].gen & 0xFFFFu);
    return SPH_OK;
}

sph_status sph_source_remove(sph_world* w, uint32_t source_h) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const int slot = edits_lookup(w->sources, source_h);
    if (slot < 0) return w->fail(SPH_ERR_INVALID, "bad source handle %u", (unsigned)source_h);
    TRY(enter(w));
    SourceRec& r = w->sources[slot];
    r.pos.release();
    r.vel.release();
    r.alive = false;
    return SPH_OK;
}

sph_status sph_fluid_read_step_edits(sph_world* w, uint32_t fluid_h, uint32_t* removed, uint32_t* emitted) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    if (removed) *removed = (uint32_t)w->fluids[fluid].step_removed;
    if (emitted) *emitted = (uint32_t)w->fluids[fluid].step_emitted;
    return SPH_OK;
}

// Fluid surface meshes (sph_surface_host.inl, DESIGN.md section 15)
sph_status sph_world_extract_surface(sph_world* w, const uint32_t* fluids, size_t n_fluids, const sph_surface_desc* desc, size_t* n_vertices,
                                     size_t* n_triangles) {
    if (!w || !desc || !n_vertices || !n_triangles || (n_fluids && !fluids)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return extract_surface(w, fluids, n_fluids, desc, nullptr, n_vertices, n_triangles);
}
void sph_surface_anisotropy_default(sph_surface_anisotropy* a) {
    if (!a) return;
    a->smoothing = 0.9f;
    a->max_ratio = 1.f;
    a->isolated_radius = 1.f;
    a->min_neighbours = 6;
}
sph_status sph_world_extract_surface_anisotropic(sph_world* w, const uint32_t* fluids, size_t n_fluids, const sph_surface_desc* desc,
                                                 const sph_surface_anisotropy* aniso, size_t* n_vertices, size_t* n_triangles) {
    if (!w || !desc || !aniso || !n_vertices || !n_triangles || (n_fluids && !fluids)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return extract_surface(w, fluids, n_fluids, desc, aniso, n_vertices, n_triangles);
}
sph_status sph_world_read_surface_ellipsoids(sph_world* w, uint32_t fluid, float* centres_xyz, float* axes, size_t cap, size_t* n) {
    if (!w || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return surface_ellipsoids(w, fluid, centres_xyz, axes, cap, nullptr, nullptr, n);
}
sph_status sph_world_map_surface_ellipsoids(sph_world* w, uint32_t fluid, const float** d_centres_xyz, const float** d_axes, size_t* n) {
    if (!w || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return surface_ellipsoids(w, fluid, nullptr, nullptr, 0, d_centres_xyz, d_axes, n);
}
sph_status sph_world_read_surface(sph_world* w, float* vertices_xyz, float* normals_xyz, size_t vcap, uint32_t* triangles, size_t tcap) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const SurfaceSet& R = w->surf.cur;
    if (vcap < R.nv || tcap < R.nt) return w->fail(SPH_ERR_INVALID, "sph_world_read_surface: caps %zu / %zu below the counts %zu / %zu", vcap, tcap, R.nv, R.nt);
    if (normals_xyz && !R.normals) return w->fail(SPH_ERR_INVALID, "sph_world_read_surface: the extraction ran without normals");
    if ((R.nv && !vertices_xyz) || (R.nt && !triangles)) return w->fail(SPH_ERR_INVALID, "sph_world_read_surface: null output");
    TRY(enter(w));
    if (R.nv) CU(cudaMemcpyAsync(vertices_xyz, R.verts.p, 3 * R.nv * sizeof(float), cudaMemcpyDeviceToHost, w->st));
    if (R.nv && normals_xyz) CU(cudaMemcpyAsync(normals_xyz, R.nrm.p, 3 * R.nv * sizeof(float), cudaMemcpyDeviceToHost, w->st));
    if (R.nt) CU(cudaMemcpyAsync(triangles, R.tris.p, 3 * R.nt * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
    CU(cudaStreamSynchronize(w->st));
    return SPH_OK;
}
sph_status sph_world_map_surface(sph_world* w, const float** d_vertices_xyz, const float** d_normals_xyz, const uint32_t** d_triangles) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const SurfaceSet& R = w->surf.cur;
    if (d_vertices_xyz) *d_vertices_xyz = R.verts.p;
    if (d_normals_xyz) *d_normals_xyz = R.normals ? R.nrm.p : nullptr;
    if (d_triangles) *d_triangles = R.tris.p;
    return SPH_OK;
}
sph_status sph_world_read_surface_field(sph_world* w, float* phi, size_t cap, float origin[3], uint32_t dims[3]) {
    if (!w || !origin || !dims) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const SurfaceSet& R = w->surf.cur;
    const size_t npts = (size_t)R.L.n[0] * R.L.n[1] * R.L.n[2];
    if (phi && cap < npts) return w->fail(SPH_ERR_INVALID, "sph_world_read_surface_field: cap %zu below the %zu lattice points", cap, npts);
    for (int a = 0; a < 3; ++a) {
        origin[a] = R.L.o[a];
        dims[a] = R.L.n[a];
    }
    if (phi && npts) {
        TRY(enter(w));
        CU(cudaMemcpyAsync(phi, R.phi.p, npts * sizeof(float), cudaMemcpyDeviceToHost, w->st));
        CU(cudaStreamSynchronize(w->st));
    }
    return SPH_OK;
}

// Diffuse particles (sph_diffuse_host.inl, DESIGN.md section 16)
void sph_diffuse_desc_default(sph_diffuse_desc* d) {
    if (!d) return;
    memset(d, 0, sizeof *d);
    d->ta_min = 2.f, d->ta_max = 8.f;
    d->wc_min = 0.5f, d->wc_max = 4.f;
    d->k_min = 0.1f, d->k_max = 2.f;
    d->k_ta = 50.f, d->k_wc = 50.f;
    d->lifetime = 2.f;
    d->k_b = 0.8f, d->k_d = 0.5f;
    d->spray_below = 6, d->bubble_above = 20;
    d->capacity = 1u << 20;
    d->seed = 0;
    for (int a = 0; a < 3; ++a) d->lo[a] = -INFINITY, d->hi[a] = INFINITY;
}
sph_status sph_world_update_diffuse(sph_world* w, const uint32_t* fluids, size_t n_fluids, const sph_diffuse_desc* desc, float dt,
                                    const float gravity[3], sph_diffuse_stats* stats) {
    if (!w || !desc || !gravity || (n_fluids && !fluids)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return update_diffuse(w, fluids, n_fluids, desc, dt, gravity, stats);
}
sph_status sph_world_read_diffuse(sph_world* w, float* pos_xyz, float* vel_xyz, uint8_t* kind, float* life, size_t cap, size_t* n) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const DiffuseSet& R = w->diffuse.cur;
    if (n) *n = R.n;
    if (!pos_xyz && !vel_xyz && !kind && !life) return SPH_OK;
    if (cap < R.n) return w->fail(SPH_ERR_INVALID, "sph_world_read_diffuse: cap %zu below the count %zu", cap, R.n);
    if (!R.n) return SPH_OK;
    TRY(enter(w));
    if (pos_xyz) CU(cudaMemcpyAsync(pos_xyz, R.pos.p, 3 * R.n * sizeof(float), cudaMemcpyDeviceToHost, w->st));
    if (vel_xyz) CU(cudaMemcpyAsync(vel_xyz, R.vel.p, 3 * R.n * sizeof(float), cudaMemcpyDeviceToHost, w->st));
    if (kind) CU(cudaMemcpyAsync(kind, R.kind.p, R.n, cudaMemcpyDeviceToHost, w->st));
    if (life) CU(cudaMemcpyAsync(life, R.life.p, R.n * sizeof(float), cudaMemcpyDeviceToHost, w->st));
    CU(cudaStreamSynchronize(w->st));
    return SPH_OK;
}
sph_status sph_world_map_diffuse(sph_world* w, const float** d_pos_xyz, const float** d_vel_xyz, const uint8_t** d_kind, const float** d_life,
                                 size_t* n) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    const DiffuseSet& R = w->diffuse.cur;
    if (d_pos_xyz) *d_pos_xyz = R.pos.p;
    if (d_vel_xyz) *d_vel_xyz = R.vel.p;
    if (d_kind) *d_kind = R.kind.p;
    if (d_life) *d_life = R.life.p;
    if (n) *n = R.n;
    return SPH_OK;
}
sph_status sph_world_clear_diffuse(sph_world* w) {
    if (!w) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    w->diffuse.cur.n = 0;
    return SPH_OK;
}

// Zero-copy read-back for renderers (testbed_plugin.rs:361-376 copies fluid.positions every frame): a DEVICE pointer to the
// fluid's positions / velocities as packed xyz f32 in ORIGINAL index order.  Valid until the next call on this world.
static sph_status fluid_map(sph_world* w, uint32_t fluid_h, bool velocities, const float** dev, size_t* n) {
    FLUID_OR_FAIL(fluid, fluid_h)
    TRY(enter(w));
    if (w->staged) {  // nothing on the device yet: build the device state (what the next step would do first)
        TRY(apply_pending_deletes(w));
        TRY(stage_up(w));
    }
    const FluidRec& f = w->fluids[fluid];
    DBuf<float>& buf = velocities ? w->map_vel : w->map_pos;
    CU(buf.ensure(3 * std::max<size_t>(w->N, 1)));
    Col<Xyz> col = fluid_col(w, Xyz{(velocities ? w->vel : w->pos)[w->cur].p}, 0, 0, (float*)nullptr);
    col.dev = buf.p;
    TRY(export_rows(w, col));
    CU(cudaStreamSynchronize(w->st));
    *dev = buf.p + 3 * f.offset;
    *n = f.n;
    return SPH_OK;
}
sph_status sph_fluid_map_positions(sph_world* w, uint32_t fluid_h, const float** dev_xyz, size_t* n) {
    if (!w || !dev_xyz || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return fluid_map(w, fluid_h, false, dev_xyz, n);
}
sph_status sph_fluid_map_velocities(sph_world* w, uint32_t fluid_h, const float** dev_xyz, size_t* n) {
    if (!w || !dev_xyz || !n) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    return fluid_map(w, fluid_h, true, dev_xyz, n);
}

// Replaces the whole particle set of a fluid: positions, velocities, velocity_changes (dfsph_solver.rs:44 — the part of the
// velocity the solver carries between steps) and caller-visible ids; volumes return to the default, IISPH pressures to 0.
// This is what a slab world's plane re-balancing needs (salva_b200/slab.py: particles move between ranks wholesale).
sph_status sph_fluid_replace_particles(sph_world* w, uint32_t fluid_h, const float* pos, const float* vel, const float* vc, const uint32_t* ids,
                                       size_t n) {
    if (!w || (n && !pos)) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    FLUID_OR_FAIL(fluid, fluid_h)
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "particles cannot be replaced from inside a coupling callback");
    TRY(enter(w));
    TRY(stage_down(w));
    FluidRec& f = w->fluids[fluid];
    std::vector<uint32_t> numbered;
    if (!ids) {
        TRY(new_ids(w, nullptr, n, &numbered));
        ids = numbered.data();
    }
    w->rows.splice(f.offset, f.n, n, pos, vel, vc, nullptr, ids);
    f.n = n;
    f.pending_delete.assign(n, 0);
    f.n_pending = 0;
    for (auto& fr : f.forces) fr.elastic.reset();  // a rest pose belongs to the particle set it was captured from
    recompute_offsets(w);
    w->slab.global_valid = false;
    return SPH_OK;
}

// ---- snapshot / restore of the state the solver carries across steps ----------------------------------------------------
// velocity_changes (dfsph_solver.rs:44, carried :704-706), the lagging dt / inv_dt (timestep_manager.rs:29-30), IISPH
// warm-start pressures (iisph_solver.rs:673-677), Becker-2009 rest pose + rotations (becker2009_elasticity.rs:84-135),
// particle ids, volumes, slab planes.  The blob restores into a world with the SAME fluids / forces / boundaries pushed in
// the same order (scene description is the caller's); particle counts may differ from the world's current ones.
namespace {
constexpr uint32_t SNAP_MAGIC = 0x53485053u;  // "SPHS"
struct SnapHeader {
    uint32_t magic, version, solver, n_fluid_slots;
    float dt, inv_dt;
    int32_t slab_lo, slab_hi;
    uint64_t n_particles, total_bytes;
};
struct SnapFluid {
    uint64_t n;
    uint32_t alive, n_forces;
};
struct SnapElastic {
    uint64_t n;
    uint32_t cap0, stride0;
};
struct Writer {
    char* p;
    size_t cap, off = 0;
    void put(const void* src, size_t bytes) {
        if (p && off + bytes <= cap) memcpy(p + off, src, bytes);
        off += bytes;
    }
};
// walks the blob layout; with a null buffer it only measures.  Device-resident pieces (elasticity) are downloaded here.
sph_status snapshot_write(sph_world* w, Writer& wr) {
    SnapHeader h;
    memset(&h, 0, sizeof h);
    h.magic = SNAP_MAGIC;
    h.version = 1;
    h.solver = (uint32_t)w->desc.solver;
    h.n_fluid_slots = (uint32_t)w->fluids.size();
    h.dt = w->dt;
    h.inv_dt = w->inv_dt;
    h.slab_lo = w->slab.lo;
    h.slab_hi = w->slab.hi;
    h.n_particles = w->N;
    const size_t header_at = wr.off;
    wr.put(&h, sizeof h);
    for (auto& f : w->fluids) {
        SnapFluid sf{f.n, f.alive ? 1u : 0u, (uint32_t)f.forces.size()};
        wr.put(&sf, sizeof sf);
    }
    for (const auto& c : w->rows.columns()) wr.put(c.p, w->N * c.row_bytes);
    for (auto& f : w->fluids)
        for (auto& fr : f.forces) {
            SnapElastic se{0, 0, 0};
            const ElasticityState* E = fr.elastic.get();
            if (fr.d.kind == SPH_FORCE_BECKER2009_ELASTICITY && E && E->n) se = SnapElastic{E->n, E->cap0, E->stride0};
            wr.put(&se, sizeof se);
            if (!se.n) continue;
            const size_t n = E->n, nl = (size_t)E->cap0 * E->stride0;
            const size_t bytes = n * sizeof(float4) + n * sizeof(uint32_t) + nl * sizeof(uint32_t) + 9 * n * sizeof(float);
            if (wr.p && wr.off + bytes <= wr.cap) {
                char* dst = wr.p + wr.off;
                CU(cudaMemcpyAsync(dst, E->pos0.p, n * sizeof(float4), cudaMemcpyDeviceToHost, w->st));
                dst += n * sizeof(float4);
                CU(cudaMemcpyAsync(dst, E->cnt0.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
                dst += n * sizeof(uint32_t);
                CU(cudaMemcpyAsync(dst, E->nbr0.p, nl * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->st));
                dst += nl * sizeof(uint32_t);
                CU(cudaMemcpyAsync(dst, E->rot.p, 9 * n * sizeof(float), cudaMemcpyDeviceToHost, w->st));
                CU(cudaStreamSynchronize(w->st));
            }
            wr.off += bytes;
        }
    if (wr.p && header_at + sizeof h <= wr.cap) {
        h.total_bytes = wr.off - header_at;
        memcpy(wr.p + header_at, &h, sizeof h);
    }
    return SPH_OK;
}
}  // namespace

sph_status sph_world_snapshot_size(sph_world* w, size_t* bytes) {
    if (!w || !bytes) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "snapshots cannot be taken from inside a coupling callback");
    TRY(enter(w));
    TRY(apply_pending_deletes(w));
    TRY(stage_down(w));  // host vectors = truth in original order; the next step re-uploads (same results: the sorted order is canonical)
    Writer wr{nullptr, 0};
    TRY(snapshot_write(w, wr));
    *bytes = wr.off;
    return SPH_OK;
}

sph_status sph_world_snapshot_save(sph_world* w, void* buffer, size_t capacity, size_t* written) {
    if (!w || !buffer) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "snapshots cannot be taken from inside a coupling callback");
    TRY(enter(w));
    TRY(apply_pending_deletes(w));
    TRY(stage_down(w));
    Writer wr{static_cast<char*>(buffer), capacity};
    TRY(snapshot_write(w, wr));
    if (written) *written = wr.off;
    if (wr.off > capacity) return w->fail(SPH_ERR_INVALID, "snapshot needs %zu bytes, buffer holds %zu", wr.off, capacity);
    return SPH_OK;
}

sph_status sph_world_snapshot_load(sph_world* w, const void* buffer, size_t length) {
    if (!w || !buffer) return SPH_ERR_INVALID;
    std::lock_guard<std::recursive_mutex> lock(g_mutex);
    if (w->in_coupling) return w->fail(SPH_ERR_INVALID, "snapshots cannot be loaded from inside a coupling callback");
    const char* p = static_cast<const char*>(buffer);
    size_t off = 0;
    auto need = [&](size_t bytes) { return off + bytes <= length; };
    SnapHeader h;
    if (!need(sizeof h)) return w->fail(SPH_ERR_INVALID, "snapshot truncated");
    memcpy(&h, p, sizeof h);
    off += sizeof h;
    if (h.magic != SNAP_MAGIC || h.version != 1) return w->fail(SPH_ERR_INVALID, "not a salva_b200 snapshot (magic %08x version %u)", h.magic, h.version);
    if (h.total_bytes > length) return w->fail(SPH_ERR_INVALID, "snapshot truncated: %llu bytes expected, %zu given", (unsigned long long)h.total_bytes, length);
    if (h.solver != (uint32_t)w->desc.solver || h.n_fluid_slots != w->fluids.size())
        return w->fail(SPH_ERR_INVALID, "snapshot was taken from a differently configured world (solver %u, %u fluids)", h.solver, h.n_fluid_slots);
    std::vector<SnapFluid> sf(h.n_fluid_slots);
    if (!need(sf.size() * sizeof(SnapFluid))) return w->fail(SPH_ERR_INVALID, "snapshot truncated");
    memcpy(sf.data(), p + off, sf.size() * sizeof(SnapFluid));
    off += sf.size() * sizeof(SnapFluid);
    uint64_t total = 0;
    for (size_t k = 0; k < sf.size(); ++k) {
        if ((sf[k].alive != 0) != w->fluids[k].alive || sf[k].n_forces != w->fluids[k].forces.size())
            return w->fail(SPH_ERR_INVALID, "snapshot fluid %zu does not match the world (alive %u, %u forces)", k, sf[k].alive, sf[k].n_forces);
        total += sf[k].n;
    }
    if (total != h.n_particles) return w->fail(SPH_ERR_INVALID, "snapshot particle counts are inconsistent");
    const size_t N = (size_t)h.n_particles;
    if (!need((3 * 3 + 2) * N * sizeof(float) + N * sizeof(uint32_t))) return w->fail(SPH_ERR_INVALID, "snapshot truncated");
    TRY(enter(w));
    TRY(stage_down(w));  // flips the world to "host vectors are the truth"; their content is replaced below
    auto take = [&](void* dst, size_t bytes) {
        memcpy(dst, p + off, bytes);
        off += bytes;
    };
    w->rows.resize(N);
    for (const auto& c : w->rows.columns()) take(c.p, N * c.row_bytes);
    for (size_t k = 0; k < sf.size(); ++k) {
        w->fluids[k].n = (size_t)sf[k].n;
        w->fluids[k].pending_delete.assign((size_t)sf[k].n, 0);
        w->fluids[k].n_pending = 0;
    }
    recompute_offsets(w);
    w->dt = h.dt;
    w->inv_dt = h.inv_dt;
    if (w->slab.active) {
        w->slab.lo = h.slab_lo;
        w->slab.hi = h.slab_hi;
        w->slab.global_valid = false;
    }
    w->Ntot = w->N;
    w->own_begin = 0;
    for (auto& f : w->fluids)
        for (auto& fr : f.forces) {
            SnapElastic se;
            if (!need(sizeof se)) return w->fail(SPH_ERR_INVALID, "snapshot truncated");
            take(&se, sizeof se);
            fr.elastic.reset();
            if (!se.n) continue;
            const size_t n = (size_t)se.n, nl = (size_t)se.cap0 * se.stride0;
            if (!need(n * sizeof(float4) + n * sizeof(uint32_t) + nl * sizeof(uint32_t) + 9 * n * sizeof(float))) return w->fail(SPH_ERR_INVALID, "snapshot truncated");
            TRY(elasticity_restore(w, fr, n, se.cap0, se.stride0, p + off));
            off += n * sizeof(float4) + n * sizeof(uint32_t) + nl * sizeof(uint32_t) + 9 * n * sizeof(float);
        }
    w->lists_valid = false;
    w->grid_ready = false;
    return SPH_OK;
}

}  // extern "C"
