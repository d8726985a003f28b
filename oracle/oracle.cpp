// oracle.cpp — CPU restatement of dimforge/salva's salva3d fluid-step path.
//
// TEST INFRASTRUCTURE ONLY.  This file is the parity oracle and the timed CPU
// baseline.  Nothing under salva_b200/ may import, link or call it; only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg do.
//
// PARITY UNPINNED: the reference (Rust, cannot be built here: no rustc/cargo,
// dependencies not vendored) ships no golden vectors or numeric tests for this
// path (SURVEY.md §4, §8c).  This restatement is therefore pinned only against
// (a) analytic known answers derived from the reference's formulas
// (tests/test_oracle_analytic.py) and (b) an independent brute-force numpy
// restatement (oracle/numpy_ref.py).  Third-party arithmetic restated from the
// published behaviour of nalgebra 0.33 (Unit::try_new_and_get, norm_squared).
//
// Structure follows the reference: hash grid -> per-particle contact lists with
// cached weight/gradient -> Jacobi passes over the lists, f32 throughout, with
// OpenMP standing in for rayon's par_iter.  Every function cites the reference
// file:line it restates (paths relative to the reference tree's src/).
//
// Build: see oracle/Makefile (g++ -O3 -march=native -fopenmp -ffp-contract=off;
// contraction is disabled because rustc never fuses a*b+c).

#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

struct V3 {
    float x, y, z;
};
static inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
static inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
static inline V3 operator*(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
static inline V3 operator/(V3 a, float s) { return {a.x / s, a.y / s, a.z / s}; }
static inline V3 operator-(V3 a) { return {-a.x, -a.y, -a.z}; }
static inline V3& operator+=(V3& a, V3 b) { a.x += b.x; a.y += b.y; a.z += b.z; return a; }
static inline V3& operator-=(V3& a, V3 b) { a.x -= b.x; a.y -= b.y; a.z -= b.z; return a; }
// nalgebra dot / norm_squared on a static 3-vector: (a0*b0 + a1*b1) + a2*b2.
static inline float dot(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
static inline float norm2(V3 a) { return dot(a, a); }
static const V3 ZERO3 = {0.f, 0.f, 0.f};
static const float F32_EPS = 1.1920929e-07f;  // f32::EPSILON (Real::default_epsilon)
static const float PI_F = 3.14159265358979323846f;

// ---- kernel/cubic_spline_kernel.rs:12-33 (dim3) ------------------------------------------------
static inline float w_scalar(float r, float h) {
    float normalizer = 8.0f / (PI_F * h * h * h);
    float q = r / h;
    float rhs;
    if (q <= 0.5f) {
        float q2 = q * q;
        rhs = 1.0f + (q2 * q - q2) * 6.0f;
    } else if (q <= 1.0f) {
        float t = 1.0f - q;
        rhs = (t * t * t) * 2.0f;  // powi(3)
    } else {
        rhs = 0.0f;
    }
    return normalizer * rhs;
}
// ---- kernel/cubic_spline_kernel.rs:55-80 -------------------------------------------------------
static inline float dw_scalar(float r, float h) {
    float normalizer = 8.0f / (PI_F * h * h * h);
    float q = r / h;
    float rhs;
    if (q > 1.0f || q <= 1.0e-5f) {
        rhs = 0.0f;
    } else if (q <= 0.5f) {
        rhs = (q * 3.0f - 2.0f) * q * 6.0f;
    } else {
        float one_q = 1.0f - q;
        rhs = -one_q * one_q * 6.0f;
    }
    return normalizer * rhs / h;
}
// ---- kernel/poly6_kernel.rs:12-40, spiky_kernel.rs:12-40, viscosity_kernel.rs:12-51 (dim3): the solver's
//      KernelDensity / KernelGradient type parameters (dfsph_solver.rs:17-20, iisph_solver.rs:17-20) ------------------
enum { KERNEL_CUBIC_SPLINE = 0, KERNEL_POLY6 = 1, KERNEL_SPIKY = 2, KERNEL_VISCOSITY = 3 };
static inline float powi(float x, int n) {  // f32::powi: repeated multiplication
    float r = 1.0f;
    for (int k = 0; k < n; ++k) r *= x;
    return r;
}
static inline float w_scalar_kind(int kind, float r, float h) {
    switch (kind) {
        case KERNEL_POLY6: {
            float normalizer = (float)(315.0 / 64.0) / (PI_F * powi(h, 9));
            return r <= h ? normalizer * powi(h * h - r * r, 3) : 0.0f;
        }
        case KERNEL_SPIKY: {
            float normalizer = 15.0f / (PI_F * powi(h, 6));
            return r <= h ? normalizer * powi(h - r, 3) : 0.0f;
        }
        case KERNEL_VISCOSITY: {
            float normalizer = 15.0f / (2.0f * PI_F * powi(h, 3));
            if (r > 0.0f && r <= h) {
                float rr_hh = r * r / (h * h);
                return normalizer * (rr_hh * (1.0f - r / (2.0f * h)) + h / (2.0f * r) - 1.0f);
            }
            return 0.0f;
        }
        default: return w_scalar(r, h);
    }
}
static inline float dw_scalar_kind(int kind, float r, float h) {
    switch (kind) {
        case KERNEL_POLY6: {
            float normalizer = (float)(315.0 / 64.0) / (PI_F * powi(h, 9));
            return r <= h ? normalizer * powi(h * h - r * r, 2) * r * -6.0f : 0.0f;
        }
        case KERNEL_SPIKY: {
            float normalizer = 15.0f / (PI_F * powi(h, 6));
            return r <= h ? -normalizer * powi(h - r, 2) * 3.0f : 0.0f;
        }
        case KERNEL_VISCOSITY: {
            float normalizer = 15.0f / (2.0f * PI_F * powi(h, 3));
            if (r > 0.0f && r <= h) {
                float rr = r * r, hh = h * h, hhh = hh * h;
                return normalizer * (-3.0f * rr / (2.0f * hhh) + 2.0f * r / hh - h / (2.0f * rr));
            }
            return 0.0f;
        }
        default: return dw_scalar(r, h);
    }
}
// ---- kernel/kernel.rs:13-15,27-29: points_apply = scalar_apply(|p1-p2|) ---------------------------
static inline float kernel_w(V3 p1, V3 p2, float h, int kind = KERNEL_CUBIC_SPLINE) { return w_scalar_kind(kind, std::sqrt(norm2(p1 - p2)), h); }
// ---- kernel/kernel.rs:18-24,32-34 + nalgebra Unit::try_new_and_get(v, eps):
//      Some((v / |v|, |v|)) iff |v|^2 > eps^2 ---------------------------------------------------------
static inline bool unit_and_norm(V3 v, V3* dir, float* n) {
    float sq = norm2(v);
    if (sq > F32_EPS * F32_EPS) {
        float nn = std::sqrt(sq);
        *dir = {v.x / nn, v.y / nn, v.z / nn};
        *n = nn;
        return true;
    }
    return false;
}
static inline V3 kernel_grad(V3 p1, V3 p2, float h, int kind = KERNEL_CUBIC_SPLINE) {
    V3 dir;
    float n;
    if (unit_and_norm(p1 - p2, &dir, &n)) return dir * dw_scalar_kind(kind, n, h);
    return ZERO3;
}

// ---- object/interaction_groups.rs:64-69 -----------------------------------------------------------
struct Groups {
    uint32_t memberships, filter;
    bool test(Groups rhs) const { return (memberships & rhs.filter) != 0 && (rhs.memberships & filter) != 0; }
};

// ---- geometry/contacts.rs:40-55 (48-byte record, as in the reference) ----------------------------
struct Contact {
    uint64_t i, i_model, j, j_model;
    float weight;
    V3 gradient;
};

struct SpinLock {
    std::atomic_flag f = ATOMIC_FLAG_INIT;
    void lock() { while (f.test_and_set(std::memory_order_acquire)) {} }
    void unlock() { f.clear(std::memory_order_release); }
};

// geometry/contacts.rs:83-87: Vec<RwLock<Vec<Contact>>>
struct ParticlesContacts {
    std::vector<std::vector<Contact>> lists;
    std::vector<SpinLock> locks;
    void reset(size_t n) {
        for (auto& l : lists) l.clear();
        if (lists.size() != n) {
            lists.resize(n);
            locks = std::vector<SpinLock>(n);
        }
    }
    void push(size_t i, const Contact& c) {
        locks[i].lock();
        lists[i].push_back(c);
        locks[i].unlock();
    }
    size_t total() const {
        size_t s = 0;
        for (auto& l : lists) s += l.size();
        return s;
    }
};

enum ForceKind { F_XSPH = 0, F_ARTIFICIAL = 1, F_AKINCI = 2, F_BECKER = 3, F_HE2014 = 4, F_WCSPH = 5, F_DFSPH_VISC = 6, F_HOST = 100 };
typedef void (*host_force_fn)(void* user, float dt, float inv_dt, float kernel_radius, size_t n, const float* pos, const float* vel, const float* dens,
                              float* acc);

struct Mat3 {
    float m[3][3];  // m[row][col]
};
static inline Mat3 mat_zero() { Mat3 r; std::memset(&r, 0, sizeof r); return r; }
static inline Mat3 mat_identity() { Mat3 r = mat_zero(); r.m[0][0] = r.m[1][1] = r.m[2][2] = 1.f; return r; }
static inline V3 mat_mul(const Mat3& a, V3 v) {
    return {(a.m[0][0] * v.x + a.m[0][1] * v.y) + a.m[0][2] * v.z, (a.m[1][0] * v.x + a.m[1][1] * v.y) + a.m[1][2] * v.z,
            (a.m[2][0] * v.x + a.m[2][1] * v.y) + a.m[2][2] * v.z};
}
static inline V3 mat_tr_mul(const Mat3& a, V3 v) {
    return {(a.m[0][0] * v.x + a.m[1][0] * v.y) + a.m[2][0] * v.z, (a.m[0][1] * v.x + a.m[1][1] * v.y) + a.m[2][1] * v.z,
            (a.m[0][2] * v.x + a.m[1][2] * v.y) + a.m[2][2] * v.z};
}
static inline V3 mat_col(const Mat3& a, int c) { return {a.m[0][c], a.m[1][c], a.m[2][c]}; }
static inline V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

struct Force {
    int kind;
    float p[8];
    host_force_fn host_fn = nullptr;  // user-defined NonPressureForce::solve (nonpressure_force.rs:10-30)
    void* host_user = nullptr;
    // Akinci2013: normals (akinci2013_surface_tension.rs:23)
    std::vector<V3> normals;
    // He2014: colors, squared colour-gradient norms (he2014_surface_tension.rs:16-17)
    std::vector<float> colors, gradcs;
    // DFSPHViscosity: betas (6x6 row-major), strain-rate targets / errors (dfsph_viscosity.rs:99-100)
    std::vector<std::array<float, 36>> betas;
    std::vector<std::array<float, 6>> sr_target, sr_error;
    uint32_t visc_iters = 0;
    float visc_err = 0.f;
    // Becker2009 state (becker2009_elasticity.rs:48-58)
    float d0 = 0, d1 = 0, d2 = 0;
    std::vector<float> volumes0;
    std::vector<V3> positions0;
    ParticlesContacts contacts0;
    std::vector<Mat3> rotations, grad_tr;
    std::vector<float> stress;  // 6 per particle: x y z w a b
};

// ---- object/fluid.rs:12-34 ------------------------------------------------------------------------
struct Fluid {
    std::vector<V3> positions, velocities, accelerations;
    std::vector<float> volumes;
    float density0;
    std::vector<uint8_t> deleted;
    size_t num_deleted = 0;
    float particle_radius;
    Groups groups;
    std::vector<Force> forces;
    size_t n() const { return positions.size(); }
    float mass(size_t i) const { return volumes[i] * density0; }  // fluid.rs:183-185
};

// ---- object/boundary.rs:11-24 ---------------------------------------------------------------------
struct Boundary {
    std::vector<V3> positions, velocities;
    std::vector<float> volumes;
    bool has_forces = false;
    std::vector<V3> forces;
    std::vector<SpinLock> flocks;
    Groups groups;
    size_t n() const { return positions.size(); }
    // boundary.rs:62-67
    void apply_force(size_t i, V3 f) {
        if (has_forces) {
            flocks[i].lock();
            forces[i] += f;
            flocks[i].unlock();
        }
    }
};

struct CellKey {
    int64_t x, y, z;
    bool operator==(const CellKey& o) const { return x == o.x && y == o.y && z == o.z; }
};
struct CellHash {  // stands in for fnv(1820); iteration order only affects f32 summation order
    size_t operator()(const CellKey& k) const {
        uint64_t h = 1469598103934665603ull ^ 1820ull;
        for (int64_t v : {k.x, k.y, k.z}) {
            h ^= (uint64_t)v;
            h *= 1099511628211ull;
        }
        return (size_t)h;
    }
};
// geometry/contacts.rs:14-19
struct GridEntry {
    uint32_t model;
    uint32_t particle;
    bool is_boundary;
};
typedef std::unordered_map<CellKey, std::vector<GridEntry>, CellHash> HGrid;

struct Timings {
    double grid_ms = 0, neighbors_ms = 0, density_ms = 0, divergence_ms = 0, nonpressure_ms = 0, pressure_ms = 0,
           integrate_ms = 0, step_ms = 0;
};

struct World {
    int solver = 0;
    float particle_radius = 0, h = 0;
    // dfsph_solver.rs:54-62 / iisph_solver.rs:48-53
    uint32_t min_pressure_iter = 1, max_pressure_iter = 50;
    float max_density_error = 0.05f;
    uint32_t min_divergence_iter = 1, max_divergence_iter = 50;
    float max_divergence_error = 0.1f;
    float omega = 0.5f;
    const size_t min_neighbors_for_divergence_solve = 20;  // dfsph_solver.rs:62 (dim3)
    // timestep_manager.rs:21-31
    float dt = 0.f, inv_dt = 0.f, total_step_size = 0.f, remaining_time = 0.f;
    int sort_contacts = 1;
    int kernel_density = KERNEL_CUBIC_SPLINE, kernel_gradient = KERNEL_CUBIC_SPLINE;  // DFSPHSolver<KernelDensity, KernelGradient>
    int force_div = -1, force_press = -1;

    std::vector<Fluid> fluids;
    std::vector<Boundary> boundaries;
    HGrid grid;
    std::vector<ParticlesContacts> ff, fb, bb;
    // DFSPH scratch dfsph_solver.rs:40-44
    std::vector<std::vector<float>> alphas, densities, predicted, divergences;
    std::vector<std::vector<V3>> vc;
    // IISPH scratch iisph_solver.rs:30-39
    std::vector<std::vector<float>> aii, pressures, next_pressures;
    std::vector<std::vector<V3>> dii, dij_pjl;
    // debug snapshot of accelerations after predict_advection
    std::vector<std::vector<V3>> dbg_acc;

    uint32_t n_div_iter = 0, n_press_iter = 0, n_div_eval = 0, n_press_eval = 0;
    float last_div_err = 0, last_dens_err = 0;
    bool edited = true;  // particles appended or deleted since the last step (the plugin scratch no longer fits them)
    Timings tm;
    std::string err;
};

static double now_ms() {
#ifdef _OPENMP
    return omp_get_wtime() * 1e3;
#else
    return 0.0;
#endif
}

// ---- geometry/hgrid.rs:41-52 ----------------------------------------------------------------------
static inline int64_t quantify(float v, float cell_width) { return (int64_t)std::floor((double)std::floor(v / cell_width)); }
static inline CellKey cell_key(V3 p, float w) { return {quantify(p.x, w), quantify(p.y, w), quantify(p.z, w)}; }

// ---- geometry/contacts.rs:133-151 (serial inserts, as the reference) ----------------------------
static void insert_to_grid(World& w) {
    w.grid.clear();
    for (size_t f = 0; f < w.fluids.size(); ++f)
        for (size_t i = 0; i < w.fluids[f].n(); ++i)
            w.grid[cell_key(w.fluids[f].positions[i], w.h)].push_back({(uint32_t)f, (uint32_t)i, false});
    for (size_t b = 0; b < w.boundaries.size(); ++b)
        for (size_t i = 0; i < w.boundaries[b].n(); ++i)
            w.grid[cell_key(w.boundaries[b].positions[i], w.h)].push_back({(uint32_t)b, (uint32_t)i, true});
}

// ---- geometry/contacts.rs:254-400 -----------------------------------------------------------------
static void contacts_for_pair_of_cells(World& w, bool same_cell, const std::vector<GridEntry>& curr,
                                       const std::vector<GridEntry>& neigh) {
    const float h2 = w.h * w.h;
    for (const GridEntry& ei : curr) {
        if (ei.is_boundary) {
            const Boundary& bi = w.boundaries[ei.model];
            for (const GridEntry& ej : neigh) {
                if (ej.is_boundary) {
                    const Boundary& bj = w.boundaries[ej.model];
                    if (ei.model != ej.model && !bi.groups.test(bj.groups)) continue;  // :276-279
                    if (norm2(bi.positions[ei.particle] - bj.positions[ej.particle]) <= h2) {
                        Contact c{ei.particle, ei.model, ej.particle, ej.model, 0.f, ZERO3};
                        w.bb[ei.model].push(ei.particle, c);
                        if (!same_cell) {  // :300-305 flip
                            Contact fc{c.j, c.j_model, c.i, c.i_model, 0.f, ZERO3};
                            w.bb[ej.model].push(ej.particle, fc);
                        }
                    }
                } else {
                    if (same_cell) continue;  // :309-312 (handled from the fluid side)
                    const Fluid& fj = w.fluids[ej.model];
                    if (!bi.groups.test(fj.groups)) continue;
                    if (norm2(bi.positions[ei.particle] - fj.positions[ej.particle]) <= h2) {
                        Contact c{ej.particle, ej.model, ei.particle, ei.model, 0.f, ZERO3};  // stored fluid side :323-335
                        w.fb[ej.model].push(ej.particle, c);
                    }
                }
            }
        } else {
            const Fluid& fi = w.fluids[ei.model];
            for (const GridEntry& ej : neigh) {
                V3 pj;
                if (ej.is_boundary) {
                    const Boundary& bj = w.boundaries[ej.model];
                    if (!fi.groups.test(bj.groups)) continue;  // :347-352
                    pj = bj.positions[ej.particle];
                } else {
                    if (ei.model != ej.model && !fi.groups.test(w.fluids[ej.model].groups)) continue;  // :355-362
                    pj = w.fluids[ej.model].positions[ej.particle];
                }
                if (norm2(fi.positions[ei.particle] - pj) <= h2) {  // :366 inclusive
                    Contact c{ei.particle, ei.model, ej.particle, ej.model, 0.f, ZERO3};
                    if (ej.is_boundary) {
                        w.fb[ei.model].push(ei.particle, c);
                    } else {
                        w.ff[ei.model].push(ei.particle, c);  // same cell: every ordered pair incl. i==i
                        if (!same_cell) {                     // :388-393 flip
                            Contact fc{c.j, c.j_model, c.i, c.i_model, 0.f, ZERO3};
                            w.ff[ej.model].push(ej.particle, fc);
                        }
                    }
                }
            }
        }
    }
}

static bool contact_less(const Contact& a, const Contact& b) {
    return a.j_model != b.j_model ? a.j_model < b.j_model : a.j < b.j;
}

// ---- geometry/contacts.rs:154-252 -----------------------------------------------------------------
static void compute_contacts(World& w) {
    w.ff.resize(w.fluids.size());
    w.fb.resize(w.fluids.size());
    w.bb.resize(w.boundaries.size());
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        w.ff[f].reset(w.fluids[f].n());
        w.fb[f].reset(w.fluids[f].n());
    }
    for (size_t b = 0; b < w.boundaries.size(); ++b) w.bb[b].reset(w.boundaries[b].n());

    static const int NB[14][3] = {{0, 0, 0},  {0, 0, 1},  {0, 1, -1}, {0, 1, 0},  {0, 1, 1}, {1, -1, -1}, {1, -1, 0},
                                  {1, -1, 1}, {1, 0, -1}, {1, 0, 0},  {1, 0, 1},  {1, 1, -1}, {1, 1, 0},  {1, 1, 1}};
    std::vector<const std::pair<const CellKey, std::vector<GridEntry>>*> cells;
    cells.reserve(w.grid.size());
    for (auto& kv : w.grid) cells.push_back(&kv);

#pragma omp parallel for schedule(dynamic, 64)
    for (long ci = 0; ci < (long)cells.size(); ++ci) {
        const CellKey& k = cells[ci]->first;
        for (int nb = 0; nb < 14; ++nb) {
            CellKey nk{k.x + NB[nb][0], k.y + NB[nb][1], k.z + NB[nb][2]};
            auto it = w.grid.find(nk);
            if (it != w.grid.end()) contacts_for_pair_of_cells(w, nb == 0, cells[ci]->second, it->second);
        }
    }
    if (w.sort_contacts) {  // determinism aid only (reference order is hash/rayon dependent)
        for (auto* sets : {&w.ff, &w.fb, &w.bb})
            for (auto& pc : *sets) {
#pragma omp parallel for schedule(static)
                for (long i = 0; i < (long)pc.lists.size(); ++i)
                    std::sort(pc.lists[i].begin(), pc.lists[i].end(), contact_less);
            }
    }
}

// ---- solver/helper.rs:9-65 ------------------------------------------------------------------------
static void evaluate_kernels(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        auto& lists = w.ff[f].lists;
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)lists.size(); ++i)
            for (Contact& c : lists[i]) {
                V3 pi = w.fluids[c.i_model].positions[c.i], pj = w.fluids[c.j_model].positions[c.j];
                c.weight = kernel_w(pi, pj, w.h, w.kernel_density);
                c.gradient = kernel_grad(pi, pj, w.h, w.kernel_gradient);
            }
        auto& blists = w.fb[f].lists;
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)blists.size(); ++i)
            for (Contact& c : blists[i]) {
                V3 pi = w.fluids[c.i_model].positions[c.i], pj = w.boundaries[c.j_model].positions[c.j];
                c.weight = kernel_w(pi, pj, w.h, w.kernel_density);
                c.gradient = kernel_grad(pi, pj, w.h, w.kernel_gradient);
            }
    }
    for (size_t b = 0; b < w.boundaries.size(); ++b) {
        auto& lists = w.bb[b].lists;
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)lists.size(); ++i)
            for (Contact& c : lists[i]) {
                V3 pi = w.boundaries[c.i_model].positions[c.i], pj = w.boundaries[c.j_model].positions[c.j];
                c.weight = kernel_w(pi, pj, w.h, w.kernel_density);
                c.gradient = kernel_grad(pi, pj, w.h, w.kernel_gradient);
            }
    }
}

// ---- dfsph_solver.rs:72-96 (dup iisph_solver.rs:66-90) ------------------------------------------
static bool compute_boundary_volumes(World& w) {
    bool ok = true;
    for (size_t b = 0; b < w.boundaries.size(); ++b) {
        Boundary& bd = w.boundaries[b];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)bd.n(); ++i) {
            float den = 0.f;
            for (const Contact& c : w.bb[b].lists[i]) den += c.weight;
            if (den == 0.f) ok = false;  // assert!(!denominator.is_zero())
            bd.volumes[i] = 1.0f / den;
        }
    }
    return ok;
}

// ---- dfsph_solver.rs:628-665 (dup iisph_solver.rs:604-641) --------------------------------------
static bool compute_densities(World& w) {
    bool ok = compute_boundary_volumes(w);
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        std::vector<float>& dens = w.densities[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)dens.size(); ++i) {
            float d = 0.f;
            for (const Contact& c : w.ff[f].lists[i]) d += w.fluids[c.j_model].mass(c.j) * c.weight;
            for (const Contact& c : w.fb[f].lists[i])
                d += w.boundaries[c.j_model].volumes[c.j] * w.fluids[c.i_model].density0 * c.weight;
            if (d == 0.f) ok = false;  // assert!(!density.is_zero())
            dens[i] = d;
        }
    }
    return ok;
}

// ---- dfsph_solver.rs:165-216 ----------------------------------------------------------------------
static void compute_alphas(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
        std::vector<float>& al = w.alphas[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)al.size(); ++i) {
            V3 grad_sum = ZERO3;
            float sq = 0.f;
            for (const Contact& c : w.ff[f].lists[i]) {
                V3 g = c.gradient * w.fluids[c.j_model].mass(c.j);
                sq += norm2(g);
                grad_sum += g;
            }
            for (const Contact& c : w.fb[f].lists[i]) {
                V3 g = c.gradient * w.boundaries[c.j_model].volumes[c.j] * fi.density0;
                sq += norm2(g);
                grad_sum += g;
            }
            float den = sq + norm2(grad_sum);
            al[i] = (den <= 1.0e-5f) ? 0.f : 1.0f / den;
        }
    }
}

// ---- dfsph_solver.rs:279-356 ----------------------------------------------------------------------
static float compute_divergences(World& w) {
    float max_error = 0.f;
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
        std::vector<float>& dv = w.divergences[f];
        float err = 0.f;
#pragma omp parallel for schedule(static) reduction(+ : err)
        for (long i = 0; i < (long)dv.size(); ++i) {
            dv[i] = 0.f;
            if (w.ff[f].lists[i].size() + w.fb[f].lists[i].size() < w.min_neighbors_for_divergence_solve) continue;
            float d = 0.f;
            for (const Contact& c : w.ff[f].lists[i]) {
                const Fluid& fj = w.fluids[c.j_model];
                V3 vi = fi.velocities[c.i] + w.vc[c.i_model][c.i];
                V3 vj = fj.velocities[c.j] + w.vc[c.j_model][c.j];
                d += dot(vi - vj, c.gradient) * fj.mass(c.j);
            }
            for (const Contact& c : w.fb[f].lists[i]) {
                V3 vi = fi.velocities[c.i] + w.vc[c.i_model][c.i];
                d += dot(vi, c.gradient) * w.boundaries[c.j_model].volumes[c.j] * fi.density0;
            }
            d = std::max(d, 0.f);
            dv[i] = d;
            err += d / fi.density0;
        }
        if (fi.n() != 0) max_error = std::max(max_error, err / (float)(double)fi.n());
    }
    return max_error;
}

// ---- dfsph_solver.rs:358-409 ----------------------------------------------------------------------
static void compute_velocity_changes_for_divergence(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& f1 = w.fluids[f];
        std::vector<V3>& vcf = w.vc[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)vcf.size(); ++i) {
            float ki = w.divergences[f][i] * w.alphas[f][i];
            V3 v = vcf[i];
            for (const Contact& c : w.ff[f].lists[i]) {
                float kj = w.divergences[c.j_model][c.j] * w.alphas[c.j_model][c.j];
                float coeff = -(ki + kj) * w.fluids[c.j_model].mass(c.j);
                v += c.gradient * coeff;
            }
            for (const Contact& c : w.fb[f].lists[i]) {
                Boundary& b2 = w.boundaries[c.j_model];
                float coeff = -ki * b2.volumes[c.j] * f1.density0;
                V3 delta = c.gradient * coeff;
                v += delta;
                b2.apply_force(c.j, delta * (-w.inv_dt * f1.mass(c.i)));
            }
            vcf[i] = v;
        }
    }
}

// ---- dfsph_solver.rs:98-162 (dup iisph_solver.rs:92-142, which returns nothing) -----------------
static float compute_predicted_densities(World& w, bool* ok) {
    float max_error = 0.f;
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
        std::vector<float>& pd = w.predicted[f];
        float err = 0.f;
        bool good = true;
#pragma omp parallel for schedule(static) reduction(+ : err)
        for (long i = 0; i < (long)pd.size(); ++i) {
            float delta = 0.f;
            for (const Contact& c : w.ff[f].lists[i]) {
                const Fluid& fj = w.fluids[c.j_model];
                V3 vi = fi.velocities[c.i] + w.vc[c.i_model][c.i];
                V3 vj = fj.velocities[c.j] + w.vc[c.j_model][c.j];
                delta += fj.mass(c.j) * dot(vi - vj, c.gradient);
            }
            for (const Contact& c : w.fb[f].lists[i]) {
                V3 vi = fi.velocities[c.i] + w.vc[c.i_model][c.i];
                V3 vj = w.boundaries[c.j_model].velocities[c.j];
                delta += w.boundaries[c.j_model].volumes[c.j] * fi.density0 * dot(vi - vj, c.gradient);
            }
            float p = w.densities[f][i] + delta * w.dt;
            if (p == 0.f) good = false;
            pd[i] = p;
            err += (p < fi.density0) ? 0.f : p / fi.density0 - 1.0f;
        }
        if (!good) *ok = false;
        if (fi.n() != 0) max_error = std::max(max_error, err / (float)(double)fi.n());
    }
    return max_error;
}

// ---- dfsph_solver.rs:218-277 ----------------------------------------------------------------------
static void compute_velocity_changes(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& f1 = w.fluids[f];
        std::vector<V3>& vcf = w.vc[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)vcf.size(); ++i) {
            float ki = (w.predicted[f][i] - f1.density0) * w.alphas[f][i];
            V3 v = vcf[i];
            for (const Contact& c : w.ff[f].lists[i]) {
                const Fluid& f2 = w.fluids[c.j_model];
                float kj = (w.predicted[c.j_model][c.j] - f2.density0) * w.alphas[c.j_model][c.j];
                float kij = std::max(ki, 0.f) + std::max(kj, 0.f);
                if (kij > 0.f) {
                    float coeff = kij * f2.mass(c.j);
                    v -= c.gradient * (coeff * w.inv_dt);
                }
            }
            if (ki > 0.f) {
                for (const Contact& c : w.fb[f].lists[i]) {
                    Boundary& b = w.boundaries[c.j_model];
                    float coeff = ki * b.volumes[c.j] * f1.density0;
                    V3 delta = c.gradient * (coeff * w.inv_dt);
                    v -= delta;
                    b.apply_force(c.j, delta * (w.inv_dt * f1.mass(c.i)));
                }
            }
            vcf[i] = v;
        }
    }
}

// ---- viscosity/xsph_viscosity.rs:30-95 ------------------------------------------------------------
static void solve_xsph(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const float cf = fc.p[0], cb = fc.p[1];
    const std::vector<float>& dens = w.densities[f];
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        V3 af = ZERO3, ab = ZERO3;
        V3 vi = fl.velocities[i];
        if (cf != 0.f)
            for (const Contact& c : w.ff[f].lists[i])
                if (c.i_model == c.j_model)
                    af += (fl.velocities[c.j] - vi) * (cf * c.weight * fl.volumes[c.j] * fl.density0 / dens[c.j]);
        if (cb != 0.f)
            for (const Contact& c : w.fb[f].lists[i]) {
                Boundary& b = w.boundaries[c.j_model];
                V3 delta = (b.velocities[c.j] - vi) * (cb * c.weight * b.volumes[c.j] * fl.density0 / dens[c.i]);
                ab += delta;
                float mi = fl.volumes[c.i] * fl.density0;
                b.apply_force(c.j, delta * (-mi * w.inv_dt));
            }
        fl.accelerations[i] += af * w.inv_dt + ab * w.inv_dt;
    }
}

// ---- viscosity/artificial_viscosity.rs:40-124 -----------------------------------------------------
static void solve_artificial(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const float cf = fc.p[0], cb = fc.p[1], alpha = fc.p[2], beta = fc.p[3], cs = fc.p[4];
    const float h = w.h;
    const std::vector<float>& dens = w.densities[f];
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        V3 facc = ZERO3, bacc = ZERO3;
        if (cf != 0.f)
            for (const Contact& c : w.ff[f].lists[i])
                if (c.i_model == c.j_model) {
                    V3 r = fl.positions[c.i] - fl.positions[c.j];
                    V3 v = fl.velocities[c.i] - fl.velocities[c.j];
                    float vr = dot(r, v);
                    if (vr < 0.f) {
                        float davg = (dens[c.i] + dens[c.j]) * 0.5f;
                        float eta2 = h * h * 0.01f;
                        float mu = h * vr / (norm2(r) + eta2);
                        facc += c.gradient * (cf * (cs * alpha * mu - beta * mu * mu) * (fl.volumes[c.j] * fl.density0 / davg));
                    }
                }
        if (cb != 0.f)
            for (const Contact& c : w.fb[f].lists[i]) {
                Boundary& b = w.boundaries[c.j_model];
                V3 r = fl.positions[c.i] - b.positions[c.j];
                V3 v = fl.velocities[c.i] - b.velocities[c.j];
                float vr = dot(r, v);
                if (vr < 0.f) {
                    float davg = dens[c.i];
                    float eta2 = h * h * 0.01f;
                    float mu = h * vr / (norm2(r) + eta2);
                    bacc += c.gradient * (cb * (cs * alpha * mu - beta * mu * mu) * (b.volumes[c.j] * fl.density0 / davg));
                    float mi = fl.volumes[c.i] * fl.density0;
                    b.apply_force(c.j, bacc * -mi);  // running sum, as the reference (:117)
                }
            }
        fl.accelerations[i] += facc + bacc;
    }
}

// ---- surface_tension/akinci2013_surface_tension.rs:71-88 (dim3) ----------------------------------
static inline float cohesion_kernel(float r, float h) {
    float normalizer = 32.0f / (PI_F * powi(h, 9));
    float coeff;
    if (r <= h / 2.0f)
        coeff = 2.0f * powi(h - r, 3) * powi(r, 3) - powi(h, 6) / 64.0f;
    else if (r <= h)
        coeff = powi(h - r, 3) * powi(r, 3);
    else
        coeff = 0.f;
    return normalizer * coeff;
}
// ---- akinci2013_surface_tension.rs:90-111 ---------------------------------------------------------
static inline float adhesion_kernel(float r, float h) {
    if (r > h / 2.0f && r <= h) {
        float normalizer = 0.007f / std::pow(h, 3.25f);
        float coeff = std::pow(std::max(-4.0f * r * r / h + 6.0f * r - 2.0f * h, 0.f), 0.25f);
        return normalizer * coeff;
    }
    return 0.f;
}
// ---- akinci2013_surface_tension.rs:37-192 ---------------------------------------------------------
static void solve_akinci(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const float gamma = fc.p[0], adh = fc.p[1], h = w.h;
    const std::vector<float>& dens = w.densities[f];
    if (fc.normals.size() != fl.n()) fc.normals.resize(fl.n(), ZERO3);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {  // compute_normals :43-68
        V3 nrm = ZERO3;
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) nrm += c.gradient * (fl.mass(c.j) / dens[c.j]);
        fc.normals[i] = nrm * h;
    }
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        V3 acc = fl.accelerations[i];
        if (gamma != 0.f)
            for (const Contact& c : w.ff[f].lists[i])
                if (c.i_model == c.j_model) {
                    V3 dpos = fl.positions[c.i] - fl.positions[c.j];
                    V3 dir;
                    float dist;
                    V3 cohesion_vec = unit_and_norm(dpos, &dir, &dist) ? dir * cohesion_kernel(dist, h) : ZERO3;
                    V3 cohesion_acc = cohesion_vec * (-gamma * fl.volumes[c.j] * fl.density0);
                    V3 curvature_acc = (fc.normals[c.i] - fc.normals[c.j]) * -gamma;
                    float kij = 2.0f * fl.density0 / (dens[c.i] + dens[c.j]);
                    acc += (curvature_acc + cohesion_acc) * kij;
                }
        if (adh != 0.f)
            for (const Contact& c : w.fb[f].lists[i]) {
                Boundary& b = w.boundaries[c.j_model];
                V3 dpos = fl.positions[c.i] - b.positions[c.j];
                V3 dir;
                float dist;
                V3 adhesion_vec = unit_and_norm(dpos, &dir, &dist) ? dir * adhesion_kernel(dist, h) : ZERO3;
                float mi = fl.volumes[c.i] * fl.density0;
                float mj = b.volumes[c.j] * fl.density0;
                V3 adhesion_acc = adhesion_vec * (adh * mj);
                acc -= adhesion_acc;
                b.apply_force(c.j, adhesion_acc * mi);
            }
        fl.accelerations[i] = acc;
    }
}

// ---- surface_tension/he2014_surface_tension.rs:31-180 --------------------------------------------
static void solve_he2014(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const float cf = fc.p[0], cb = fc.p[1];
    const std::vector<float>& dens = w.densities[f];
    if (fc.gradcs.size() != fl.n()) {  // init :31-38
        fc.gradcs.resize(fl.n(), 0.f);
        fc.colors.resize(fl.n(), 0.f);
    }
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {  // compute_colors :40-75
        float color = 0.f;
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) color += c.weight * fl.mass(c.j) / dens[c.j];
        for (const Contact& c : w.fb[f].lists[i]) color += c.weight * w.boundaries[c.j_model].volumes[c.j];
        fc.colors[i] = color;
    }
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {  // compute_gradc :77-105
        V3 gradc = ZERO3;
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) gradc += c.gradient * fc.colors[c.j] * fl.mass(c.j) / dens[c.j];
        V3 q = gradc / fc.colors[i];
        fc.gradcs[i] = norm2(q);
    }
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {  // forces :131-178
        V3 acc = fl.accelerations[i];
        const float mi = fl.volumes[i] * fl.density0;
        if (cf != 0.f)
            for (const Contact& c : w.ff[f].lists[i])
                if (c.i_model == c.j_model) {
                    float mj = fl.volumes[c.j] * fl.density0;
                    float gradsum = fc.gradcs[c.i] + fc.gradcs[c.j];
                    V3 fo = c.gradient * (mi / dens[c.i] * mj / dens[c.j] * gradsum / 2.0f);
                    acc += fo * (cf / (2.0f * mi));
                }
        if (cb != 0.f)
            for (const Contact& c : w.fb[f].lists[i]) {
                Boundary& b = w.boundaries[c.j_model];
                float mj = b.volumes[c.j] * fl.density0;
                float gradsum = fc.gradcs[c.i];
                V3 fo = c.gradient * (mi / dens[c.i] * mj / fl.density0 * gradsum * cb * 0.25f);
                acc += fo / mi;
                b.apply_force(c.j, fo * -1.0f);
            }
        fl.accelerations[i] = acc;
    }
}

// ---- nalgebra 0.33 (crates.io dependency, build/salva3d/Cargo.toml:42; not vendored): linalg/lu.rs ------------------
// LU::new — partial pivoting (icamax = FIRST largest |.| of the column), multipliers scaled by the RECIPROCAL of the
// pivot (`coeffs *= inv_diag`), trailing update `down[:,k] = (-pivot_row[k]) * coeffs + down[:,k]` (axpy, no FMA);
// determinant = product of the diagonal times the permutation sign; try_inverse = permute identity, forward
// substitution with unit diagonal (column axpy form), back substitution (`coeff = b[i] / diag`), None on a zero pivot.
struct LU6 {
    float a[6][6];
    int swaps[6][2];
    int nswaps = 0;
};
static void lu6_new(const float m[6][6], LU6& lu) {
    std::memcpy(lu.a, m, sizeof lu.a);
    lu.nswaps = 0;
    for (int i = 0; i < 6; ++i) {
        int piv = i;
        float best = std::fabs(lu.a[i][i]);
        for (int r = i + 1; r < 6; ++r)
            if (std::fabs(lu.a[r][i]) > best) {
                best = std::fabs(lu.a[r][i]);
                piv = r;
            }
        float diag = lu.a[piv][i];
        if (diag == 0.f) continue;
        if (piv != i) {
            lu.swaps[lu.nswaps][0] = i;
            lu.swaps[lu.nswaps][1] = piv;
            lu.nswaps++;
            for (int c = 0; c < 6; ++c) std::swap(lu.a[i][c], lu.a[piv][c]);
        }
        float inv_diag = 1.0f / diag;
        for (int r = i + 1; r < 6; ++r) lu.a[r][i] *= inv_diag;
        for (int k = i + 1; k < 6; ++k) {
            float mp = -lu.a[i][k];
            for (int r = i + 1; r < 6; ++r) lu.a[r][k] = mp * lu.a[r][i] + lu.a[r][k];
        }
    }
}
static float lu6_determinant(const LU6& lu) {
    float res = 1.f;
    for (int i = 0; i < 6; ++i) res *= lu.a[i][i];
    return (lu.nswaps & 1) ? res * -1.f : res * 1.f;
}
static bool lu6_try_inverse(const LU6& lu, float out[6][6]) {
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) out[r][c] = r == c ? 1.f : 0.f;
    for (int sidx = 0; sidx < lu.nswaps; ++sidx)
        for (int c = 0; c < 6; ++c) std::swap(out[lu.swaps[sidx][0]][c], out[lu.swaps[sidx][1]][c]);
    for (int k = 0; k < 6; ++k) {  // solve_lower_triangular_with_diag_mut(b, 1)
        for (int i = 0; i < 5; ++i) {
            float coeff = out[i][k] / 1.0f;
            for (int r = i + 1; r < 6; ++r) out[r][k] = (-coeff) * lu.a[r][i] + out[r][k];
        }
    }
    for (int k = 0; k < 6; ++k) {  // solve_upper_triangular_mut
        for (int i = 5; i >= 0; --i) {
            float diag = lu.a[i][i];
            if (diag == 0.f) return false;
            float coeff = out[i][k] / diag;
            out[i][k] = coeff;
            for (int r = 0; r < i; ++r) out[r][k] = (-coeff) * lu.a[r][i] + out[r][k];
        }
    }
    return true;
}

// ---- viscosity/dfsph_viscosity.rs -----------------------------------------------------------------
// compute_gradient_matrix :59-82 (6x3, dim3)
static inline void visc_gradient_matrix(V3 g, float m[6][3]) {
    const float r[6][3] = {{g.x * 2.f, 0.f, 0.f}, {0.f, g.y * 2.f, 0.f}, {0.f, 0.f, g.z * 2.f}, {g.y, g.x, 0.f}, {g.z, 0.f, g.x}, {0.f, g.z, g.y}};
    std::memcpy(m, r, sizeof r);
}
// compute_strain_rate :38-57
static inline void visc_strain_rate(V3 g, V3 v, float out[6]) {
    out[0] = 2.f * v.x * g.x;
    out[1] = 2.f * v.y * g.y;
    out[2] = 2.f * v.z * g.z;
    out[3] = v.x * g.y + v.y * g.x;
    out[4] = v.x * g.z + v.z * g.x;
    out[5] = v.y * g.z + v.z * g.y;
}
// compute_betas :133-201
static void visc_compute_betas(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const std::vector<float>& dens = w.densities[f];
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        float grad_sum[6][3] = {}, sq[6][6] = {};
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) {
                float mat[6][3], gi[6][3];
                visc_gradient_matrix(c.gradient, mat);
                const float s = fl.mass(c.j) / (2.0f * dens[c.i]);
                for (int r = 0; r < 6; ++r)
                    for (int k = 0; k < 3; ++k) gi[r][k] = mat[r][k] * s;
                for (int r = 0; r < 6; ++r)
                    for (int cc = 0; cc < 6; ++cc) {
                        float e = gi[r][0] * gi[cc][0];
                        e += gi[r][1] * gi[cc][1];
                        e += gi[r][2] * gi[cc][2];
                        sq[r][cc] += e / dens[c.i];
                    }
                for (int r = 0; r < 6; ++r)
                    for (int k = 0; k < 3; ++k) grad_sum[r][k] += gi[r][k];
            }
        float den[6][6];
        for (int r = 0; r < 6; ++r)
            for (int cc = 0; cc < 6; ++cc) {
                float e = grad_sum[r][0] * grad_sum[cc][0];
                e += grad_sum[r][1] * grad_sum[cc][1];
                e += grad_sum[r][2] * grad_sum[cc][2];
                den[r][cc] = sq[r][cc] + e / dens[i];
            }
        float inv_diag[6];  // "Preconditionner" :162-174 (only the first SPATIAL_DIM columns are scaled)
        for (int k = 0; k < 6; ++k) inv_diag[k] = std::fabs(den[k][k]) < 1.0e-6f ? 1.f : 1.f / den[k][k];
        for (int cc = 0; cc < 3; ++cc)
            for (int r = 0; r < 6; ++r) den[r][cc] *= inv_diag[r];
        LU6 lu;  // :185-191 (the dim3 block :176-184 is overwritten by this one)
        lu6_new(den, lu);
        float inv[6][6];
        std::array<float, 36>& beta = fc.betas[i];
        if (std::fabs(lu6_determinant(lu)) < 1.0e-6f || !lu6_try_inverse(lu, inv)) {
            beta.fill(0.f);
        } else {
            for (int r = 0; r < 6; ++r)
                for (int cc = 0; cc < 6; ++cc) beta[r * 6 + cc] = inv[r][cc];
        }
        for (int cc = 0; cc < 3; ++cc)  // :193-196
            for (int r = 0; r < 6; ++r) beta[r * 6 + cc] *= inv_diag[cc];
    }
}
// compute_strain_rates :203-252
static float visc_compute_strain_rates(World& w, size_t f, Force& fc, bool compute_error) {
    Fluid& fl = w.fluids[f];
    const std::vector<float>& dens = w.densities[f];
    const float visc = fc.p[0];
    std::vector<float> per(fl.n(), 0.f);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        float rate[6] = {};
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) {
                V3 v_i = fl.velocities[c.i] + fl.accelerations[c.i] * w.dt;
                V3 v_j = fl.velocities[c.j] + fl.accelerations[c.j] * w.dt;
                float r6[6];
                visc_strain_rate(c.gradient, v_j - v_i, r6);
                const float s = fl.mass(c.j) / (2.0f * dens[c.i]);
                for (int k = 0; k < 6; ++k) rate[k] += r6[k] * s;
            }
        if (compute_error) {
            float l1 = 0.f;
            for (int k = 0; k < 6; ++k) {
                fc.sr_error[i][k] = rate[k] - fc.sr_target[i][k];
                l1 += std::fabs(fc.sr_error[i][k]);
            }
            per[i] = l1 / 6.0f;
        } else {
            for (int k = 0; k < 6; ++k) fc.sr_target[i][k] = rate[k] * (1.0f - visc);
        }
    }
    float err = 0.f;  // par_reduce_sum: f32 sum (order unspecified in the reference)
    for (size_t i = 0; i < fl.n(); ++i) err += per[i];
    return fl.n() ? std::max(0.f, err / (float)fl.n()) : 0.f;
}
// compute_accelerations :254-289
static void visc_compute_accelerations(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const std::vector<float>& dens = w.densities[f];
    std::vector<std::array<float, 6>> u(fl.n());
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {  // u = betas * error / rho^2 (per particle; the reference recomputes it per contact)
        const std::array<float, 36>& b = fc.betas[i];
        for (int r = 0; r < 6; ++r) {
            float e = b[r * 6 + 0] * fc.sr_error[i][0];
            for (int k = 1; k < 6; ++k) e += b[r * 6 + k] * fc.sr_error[i][k];
            u[i][r] = e / (dens[i] * dens[i]);
        }
    }
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        V3 acc = fl.accelerations[i];
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) {
                float co[6];
                const float hm = fl.volumes[c.j] * fl.density0 / 2.0f;
                for (int k = 0; k < 6; ++k) co[k] = (u[c.i][k] + u[c.j][k]) * hm;
                const V3 g = c.gradient;  // gradient.tr_mul(&coeff): sequential dot products over the 6 rows
                V3 t = {(g.x * 2.f) * co[0] + g.y * co[3] + g.z * co[4], (g.y * 2.f) * co[1] + g.x * co[3] + g.z * co[5],
                        (g.z * 2.f) * co[2] + g.x * co[4] + g.y * co[5]};
                acc += t * (fl.volumes[c.i] * fl.density0 * w.inv_dt);
            }
        fl.accelerations[i] = acc;
    }
}
// DFSPHViscosity::solve :292-324 (p[0] = viscosity coefficient, p[1] = min iter, p[2] = max iter, p[3] = max error)
static void solve_dfsph_viscosity(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    if (fc.betas.size() != fl.n()) {  // init :126-131
        std::array<float, 36> z36;
        z36.fill(0.f);
        std::array<float, 6> z6;
        z6.fill(0.f);
        fc.betas.resize(fl.n(), z36);
        fc.sr_target.resize(fl.n(), z6);
        fc.sr_error.resize(fl.n(), z6);
    }
    const uint32_t min_iter = (uint32_t)fc.p[1], max_iter = (uint32_t)fc.p[2];
    const float max_error = fc.p[3];
    visc_compute_betas(w, f, fc);
    visc_compute_strain_rates(w, f, fc, false);
    fc.visc_iters = 0;
    for (uint32_t i = 0; i < max_iter; ++i) {
        float avg_err = visc_compute_strain_rates(w, f, fc, true);
        fc.visc_err = avg_err;
        if (avg_err <= max_error && i >= min_iter) break;
        visc_compute_accelerations(w, f, fc);
        fc.visc_iters++;
    }
}

// ---- surface_tension/wcsph_surface_tension.rs:29-86 ---------------------------------------------
// Only the fluid term: the reference's boundary loop (:66-83) iterates fluid_fluid_contacts and indexes
// `boundaries[c.j_model].positions[c.j]` with FLUID ids (out-of-bounds panic or garbage), so a non-zero boundary
// coefficient is rejected at push time by both this restatement and the CUDA path.
static void solve_wcsph(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const float cf = fc.p[0];
    if (cf == 0.f) return;
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)fl.n(); ++i) {
        V3 acc = fl.accelerations[i];
        for (const Contact& c : w.ff[f].lists[i])
            if (c.i_model == c.j_model) {
                V3 dpos = fl.positions[c.i] - fl.positions[c.j];
                acc += dpos * (-cf * c.weight * fl.volumes[c.j] * fl.density0 / (fl.volumes[c.i] * fl.density0));
            }
        fl.accelerations[i] = acc;
    }
}

// ---- geometry/contacts.rs:403-446 + hgrid.rs:93-103 (27-cell stencil, self included) -----------
static void compute_self_contacts(float h, const Fluid& fl, ParticlesContacts& pc) {
    pc.reset(fl.n());
    std::unordered_map<CellKey, std::vector<uint32_t>, CellHash> grid;
    for (size_t i = 0; i < fl.n(); ++i) grid[cell_key(fl.positions[i], h)].push_back((uint32_t)i);
    const float h2 = h * h;
    for (auto& kv : grid) {
        for (int dz = -1; dz <= 1; ++dz)
            for (int dy = -1; dy <= 1; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                    auto it = grid.find({kv.first.x + dx, kv.first.y + dy, kv.first.z + dz});
                    if (it == grid.end()) continue;
                    for (uint32_t pi : kv.second)
                        for (uint32_t pj : it->second)
                            if (norm2(fl.positions[pi] - fl.positions[pj]) <= h2)
                                pc.lists[pi].push_back({pi, 0, pj, 0, 0.f, ZERO3});
                }
    }
    for (auto& l : pc.lists) std::sort(l.begin(), l.end(), contact_less);
}

// ---- nalgebra 0.33 Rotation3::from_matrix_eps(m, eps, max_iter, guess) ---------------------------
// Restated from the published algorithm ("A Robust Method to Extract the Rotational Part of
// Deformations", Müller et al. 2016) as implemented by nalgebra 0.33 geometry/rotation_specialization.rs:
//   for _ in 0..max_iter { axis = Σ_c R.col(c) × M.col(c); denom = Σ_c R.col(c)·M.col(c);
//       axisangle = axis / (|denom| + eps); if |axisangle|^2 > eps^2 { R = Rot(axisangle) * R } else break }
// (the later "perturbation at stationary points" refinement is omitted: it only triggers for
//  degenerate inputs).  PARITY UNPINNED at this boundary.
static Mat3 rot_from_scaled_axis(V3 aa) {
    float angle = std::sqrt(norm2(aa));
    if (angle == 0.f) return mat_identity();
    V3 u = {aa.x / angle, aa.y / angle, aa.z / angle};
    float s = std::sin(angle), c = std::cos(angle), t = 1.f - c;
    Mat3 r;
    r.m[0][0] = u.x * u.x * t + c;       r.m[0][1] = u.x * u.y * t - u.z * s; r.m[0][2] = u.x * u.z * t + u.y * s;
    r.m[1][0] = u.x * u.y * t + u.z * s; r.m[1][1] = u.y * u.y * t + c;       r.m[1][2] = u.y * u.z * t - u.x * s;
    r.m[2][0] = u.x * u.z * t - u.y * s; r.m[2][1] = u.y * u.z * t + u.x * s; r.m[2][2] = u.z * u.z * t + c;
    return r;
}
static Mat3 mat_mat(const Mat3& a, const Mat3& b) {
    Mat3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.m[i][j] = (a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j]) + a.m[i][2] * b.m[2][j];
    return r;
}
static Mat3 rotation_from_matrix_eps(const Mat3& m, float eps, int max_iter, Mat3 guess) {
    Mat3 rot = guess;
    for (int it = 0; it < max_iter; ++it) {
        V3 axis = cross(mat_col(rot, 0), mat_col(m, 0)) + cross(mat_col(rot, 1), mat_col(m, 1)) +
                  cross(mat_col(rot, 2), mat_col(m, 2));
        float denom = dot(mat_col(rot, 0), mat_col(m, 0)) + dot(mat_col(rot, 1), mat_col(m, 1)) +
                      dot(mat_col(rot, 2), mat_col(m, 2));
        V3 aa = axis * (1.0f / (std::fabs(denom) + eps));
        if (norm2(aa) > eps * eps)
            rot = mat_mat(rot_from_scaled_axis(aa), rot);
        else
            break;
    }
    return rot;
}

// becker2009_elasticity.rs:27-37 sym_mat_mul_vec: stress = (x y z w a b)
static inline V3 sym_mul(const float* s, V3 v) {
    return {(s[0] * v.x + s[3] * v.y) + s[4] * v.z, (s[3] * v.x + s[1] * v.y) + s[5] * v.z,
            (s[4] * v.x + s[5] * v.y) + s[2] * v.z};
}

// ---- elasticity/becker2009_elasticity.rs:84-334 ---------------------------------------------------
static void solve_becker(World& w, size_t f, Force& fc) {
    Fluid& fl = w.fluids[f];
    const float h = w.h;
    const size_t n = fl.n();
    const bool nonlinear = fc.p[2] != 0.f;
    if (fc.positions0.size() != n) {  // init :84-113
        float E = fc.p[0], nu = fc.p[1];
        fc.d0 = (E * (1.f - nu)) / ((1.f + nu) * (1.f - 2.f * nu));  // :15-25
        fc.d1 = (E * nu) / ((1.f + nu) * (1.f - 2.f * nu));
        fc.d2 = (E * (1.f - 2.f * nu)) / (2.f * (1.f + nu) * (1.f - 2.f * nu));
        fc.positions0 = fl.positions;
        fc.volumes0.resize(n, 0.f);  // NOTE: resize keeps old values, as Vec::resize does
        fc.rotations.resize(n, mat_identity());
        fc.grad_tr.resize(n, mat_identity());
        fc.stress.resize(6 * n, 0.f);
        compute_self_contacts(h, fl, fc.contacts0);
        for (auto& l : fc.contacts0.lists)
            for (Contact& c : l) {
                V3 p1 = fc.positions0[c.i], p2 = fc.positions0[c.j];
                c.weight = kernel_w(p1, p2, h);
                c.gradient = kernel_grad(p1, p2, h);
                fc.volumes0[c.i] += fl.mass(c.j) * c.weight;
                fc.volumes0[c.j] += fl.mass(c.i) * c.weight;
            }
        for (size_t i = 0; i < n; ++i) fc.volumes0[i] = fl.mass(i) / fc.volumes0[i];
    }
    // compute_rotations :115-137
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; ++i) {
        Mat3 apq = mat_zero();
        for (const Contact& c : fc.contacts0.lists[i]) {
            V3 p = fl.positions[c.j] - fl.positions[c.i];
            V3 p0 = fc.positions0[c.j] - fc.positions0[c.i];
            float coeff = c.weight * fl.mass(c.j);
            V3 q = p0 * coeff;
            apq.m[0][0] += p.x * q.x; apq.m[0][1] += p.x * q.y; apq.m[0][2] += p.x * q.z;
            apq.m[1][0] += p.y * q.x; apq.m[1][1] += p.y * q.y; apq.m[1][2] += p.y * q.z;
            apq.m[2][0] += p.z * q.x; apq.m[2][1] += p.z * q.y; apq.m[2][2] += p.z * q.z;
        }
        fc.rotations[i] = rotation_from_matrix_eps(apq, F32_EPS, 20, fc.rotations[i]);
    }
    // compute_stresses :139-262
    const float k = 0.564f;  // sic: the constant named _0_5 in the reference (:141)
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; ++i) {
        Mat3 g = mat_zero();
        for (const Contact& c : fc.contacts0.lists[i]) {
            V3 p = fl.positions[c.j] - fl.positions[c.i];
            V3 p0 = fc.positions0[c.j] - fc.positions0[c.i];
            V3 u = mat_tr_mul(fc.rotations[c.i], p) - p0;  // inverse_transform_vector
            V3 a = c.gradient * fc.volumes0[c.j];
            g.m[0][0] += a.x * u.x; g.m[0][1] += a.x * u.y; g.m[0][2] += a.x * u.z;
            g.m[1][0] += a.y * u.x; g.m[1][1] += a.y * u.y; g.m[1][2] += a.y * u.z;
            g.m[2][0] += a.z * u.x; g.m[2][1] += a.z * u.y; g.m[2][2] += a.z * u.z;
        }
        fc.grad_tr[i] = g;
        float* s = &fc.stress[6 * i];
        if (nonlinear) {
            Mat3 j = g;
            j.m[0][0] += 1.f; j.m[1][1] += 1.f; j.m[2][2] += 1.f;
            Mat3 jt;
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) jt.m[a][b] = j.m[b][a];
            Mat3 jjt = mat_mat(j, jt);
            V3 e = {jjt.m[0][0] - 1.f, jjt.m[1][1] - 1.f, jjt.m[2][2] - 1.f};
            V3 s012 = {(fc.d0 * e.x + fc.d1 * e.y) + fc.d1 * e.z, (fc.d1 * e.x + fc.d0 * e.y) + fc.d1 * e.z,
                       (fc.d1 * e.x + fc.d1 * e.y) + fc.d0 * e.z};
            s[0] = s012.x * k; s[1] = s012.y * k; s[2] = s012.z * k;
            s[3] = jjt.m[1][0] * k * fc.d2; s[4] = jjt.m[2][0] * k * fc.d2; s[5] = jjt.m[2][1] * k * fc.d2;
        } else {
            V3 e = {g.m[0][0], g.m[1][1], g.m[2][2]};
            s[0] = (fc.d0 * e.x + fc.d1 * e.y) + fc.d1 * e.z;
            s[1] = (fc.d1 * e.x + fc.d0 * e.y) + fc.d1 * e.z;
            s[2] = (fc.d1 * e.x + fc.d1 * e.y) + fc.d0 * e.z;
            s[3] = (g.m[1][0] + g.m[0][1]) * k * fc.d2;
            s[4] = (g.m[2][0] + g.m[0][2]) * k * fc.d2;
            s[5] = (g.m[1][2] + g.m[2][1]) * k * fc.d2;
        }
    }
    // forces :268-334
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; ++i) {
        V3 acc = fl.accelerations[i];
        for (const Contact& c : fc.contacts0.lists[i]) {
            V3 d_ij = c.gradient * fc.volumes0[c.j];
            V3 sd_ij = sym_mul(&fc.stress[6 * c.i], d_ij);
            V3 d_ji = c.gradient * (-fc.volumes0[c.i]);
            V3 sd_ji = sym_mul(&fc.stress[6 * c.j], d_ji);
            V3 f_ji, f_ij;
            if (nonlinear) {
                f_ji = (sd_ij + mat_mul(fc.grad_tr[c.i], sd_ij)) * -fc.volumes0[c.i];
                f_ij = (sd_ji + mat_mul(fc.grad_tr[c.j], sd_ji)) * -fc.volumes0[c.j];
            } else {
                f_ji = sd_ij * -fc.volumes0[c.i];
                f_ij = sd_ji * -fc.volumes0[c.j];
            }
            V3 force = (mat_mul(fc.rotations[c.j], f_ij) - mat_mul(fc.rotations[c.i], f_ji)) * 0.5f;
            float mi = fl.volumes[i] * fl.density0;
            acc += V3{force.x / mi, force.y / mi, force.z / mi};
        }
        fl.accelerations[i] = acc;
    }
}

// ---- dfsph_solver.rs:565-604 (dup iisph_solver.rs:541-580) --------------------------------------
static void predict_advection(World& w, V3 gravity) {
    for (Fluid& fl : w.fluids) {
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fl.n(); ++i) fl.accelerations[i] += gravity;
    }
    for (size_t f = 0; f < w.fluids.size(); ++f)
        for (Force& fc : w.fluids[f].forces) {
            switch (fc.kind) {
                case F_XSPH: solve_xsph(w, f, fc); break;
                case F_ARTIFICIAL: solve_artificial(w, f, fc); break;
                case F_AKINCI: solve_akinci(w, f, fc); break;
                case F_BECKER: solve_becker(w, f, fc); break;
                case F_HE2014: solve_he2014(w, f, fc); break;
                case F_WCSPH: solve_wcsph(w, f, fc); break;
                case F_DFSPH_VISC: solve_dfsph_viscosity(w, f, fc); break;
                case F_HOST: {
                    Fluid& fl = w.fluids[f];
                    fc.host_fn(fc.host_user, w.dt, w.inv_dt, w.h, fl.n(), &fl.positions[0].x, &fl.velocities[0].x, w.densities[f].data(),
                               &fl.accelerations[0].x);
                    break;
                }
            }
        }
    w.dbg_acc.resize(w.fluids.size());
    for (size_t f = 0; f < w.fluids.size(); ++f) w.dbg_acc[f] = w.fluids[f].accelerations;
}

// ---- timestep_manager.rs:76-88 --------------------------------------------------------------------
static void timestep_advance(World& w) {
    float substep = w.total_step_size;
    w.dt = substep;
    w.inv_dt = (substep == 0.f) ? 0.f : 1.0f / substep;
    w.remaining_time -= w.dt;
}

// ---- dfsph_solver.rs:505-518 (dup iisph_solver.rs:458-471) --------------------------------------
static void integrate_and_clear_accelerations(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        Fluid& fl = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fl.n(); ++i) {
            w.vc[f][i] += fl.accelerations[i] * w.dt;
            fl.accelerations[i] = ZERO3;
        }
    }
}

// ---- dfsph_solver.rs:667-708 ----------------------------------------------------------------------
static bool dfsph_step(World& w, V3 gravity) {
    bool ok = true;
    double t0 = now_ms();
    compute_alphas(w);
    double t1 = now_ms();
    w.tm.density_ms += t1 - t0;
    // divergence_solve :466-503
    w.n_div_iter = w.n_div_eval = 0;
    for (uint32_t i = 0; i < (w.force_div >= 0 ? (uint32_t)w.force_div + 1 : w.max_divergence_iter); ++i) {
        float avg = compute_divergences(w);
        w.n_div_eval++;
        w.last_div_err = avg;
        float max_err = w.max_divergence_error * w.inv_dt * 0.01f;
        if (w.force_div >= 0) {
            if ((int)i >= w.force_div) break;
        } else if (avg <= max_err && i >= w.min_divergence_iter)
            break;
        compute_velocity_changes_for_divergence(w);
        w.n_div_iter++;
    }
    double t2 = now_ms();
    w.tm.divergence_ms += t2 - t1;
    // update_velocities :422-430 and zero vc :689-691
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        Fluid& fl = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fl.n(); ++i) {
            fl.velocities[i] += w.vc[f][i];
            w.vc[f][i] = ZERO3;
        }
    }
    double t3 = now_ms();
    predict_advection(w, gravity);
    double t4 = now_ms();
    w.tm.nonpressure_ms += t4 - t3;
    timestep_advance(w);
    integrate_and_clear_accelerations(w);
    double t5 = now_ms();
    // pressure_solve :432-464
    w.n_press_iter = w.n_press_eval = 0;
    for (uint32_t i = 0; i < (w.force_press >= 0 ? (uint32_t)w.force_press + 1 : w.max_pressure_iter); ++i) {
        float avg = compute_predicted_densities(w, &ok);
        w.n_press_eval++;
        w.last_dens_err = avg;
        if (w.force_press >= 0) {
            if ((int)i >= w.force_press) break;
        } else if (avg <= w.max_density_error && i >= w.min_pressure_iter)
            break;
        compute_velocity_changes(w);
        w.n_press_iter++;
    }
    double t6 = now_ms();
    w.tm.pressure_ms += t6 - t5;
    // update_positions :411-420
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        Fluid& fl = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fl.n(); ++i) fl.positions[i] += (fl.velocities[i] + w.vc[f][i]) * w.dt;
    }
    w.tm.integrate_ms += (t3 - t2) + (t5 - t4) + (now_ms() - t6);
    return ok;
}

// ---- iisph_solver.rs:144-186 ----------------------------------------------------------------------
static void iisph_compute_dii(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fi.n(); ++i) {
            V3 d = ZERO3;
            float rhoi = w.densities[f][i];
            float factor = -w.dt * w.dt / (rhoi * rhoi);
            for (const Contact& c : w.ff[f].lists[i]) d += c.gradient * (w.fluids[c.j_model].mass(c.j) * factor);
            for (const Contact& c : w.fb[f].lists[i])
                d += c.gradient * (w.boundaries[c.j_model].volumes[c.j] * fi.density0 * factor);
            w.dii[f][i] = d;
        }
    }
}
// ---- iisph_solver.rs:188-233 ----------------------------------------------------------------------
static void iisph_compute_aii(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fi.n(); ++i) {
            float a = 0.f;
            float rhoi = w.densities[f][i];
            float mi = fi.mass(i);
            float factor = w.dt * w.dt * mi / (rhoi * rhoi);
            for (const Contact& c : w.ff[f].lists[i]) {
                float mj = w.fluids[c.j_model].mass(c.j);
                V3 dji = c.gradient * factor;
                a += mj * dot(w.dii[f][c.i] - dji, c.gradient);
            }
            for (const Contact& c : w.fb[f].lists[i]) {
                float mj = w.boundaries[c.j_model].volumes[c.j] * fi.density0;
                V3 dji = c.gradient * factor;
                a += mj * dot(w.dii[f][c.i] - dji, c.gradient);
            }
            w.aii[f][i] = a;
        }
    }
}
// ---- iisph_solver.rs:235-268 ----------------------------------------------------------------------
static void iisph_compute_dij_pjl(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)w.fluids[f].n(); ++i) {
            V3 d = ZERO3;
            for (const Contact& c : w.ff[f].lists[i]) {
                float rhoj = w.densities[c.j_model][c.j];
                float mj = w.fluids[c.j_model].mass(c.j);
                float pj = w.pressures[c.j_model][c.j];
                d += c.gradient * (-mj * pj / (rhoj * rhoj));
            }
            w.dij_pjl[f][i] = d * (w.dt * w.dt);
        }
    }
}
// ---- iisph_solver.rs:270-353 ----------------------------------------------------------------------
static float iisph_compute_next_pressures(World& w) {
    float max_error = 0.f;
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
        float err = 0.f;
#pragma omp parallel for schedule(static) reduction(+ : err)
        for (long i = 0; i < (long)fi.n(); ++i) {
            float aii = w.aii[f][i];
            float np = 0.f;
            if (std::fabs(aii) > 1.0e-9f) {
                float sum = 0.f;
                float pi = w.pressures[f][i];
                float mi = fi.mass(i);
                float rhoi = w.densities[f][i];
                float derr = fi.density0 - w.predicted[f][i];
                for (const Contact& c : w.ff[f].lists[i]) {
                    float mj = w.fluids[c.j_model].mass(c.j);
                    V3 dji = c.gradient * (w.dt * w.dt * mi / (rhoi * rhoi));
                    V3 factor = w.dij_pjl[c.i_model][c.i] - w.dii[c.j_model][c.j] * w.pressures[c.j_model][c.j] -
                                (w.dij_pjl[c.j_model][c.j] - dji * pi);
                    sum += mj * dot(factor, c.gradient);
                }
                for (const Contact& c : w.fb[f].lists[i]) {
                    float mj = w.boundaries[c.j_model].volumes[c.j] * fi.density0;
                    sum += mj * dot(w.dij_pjl[c.i_model][c.i], c.gradient);
                }
                np = (1.0f - w.omega) * pi + w.omega * (derr - sum) / aii;
                if (np > 0.f) {
                    err += (-sum - aii * np) / fi.density0;
                } else {
                    np = 0.f;
                }
            }
            w.next_pressures[f][i] = np;
        }
        if (fi.n() != 0) max_error = std::max(max_error, err / (float)(double)fi.n());
    }
    return max_error;
}
// ---- iisph_solver.rs:355-404 ----------------------------------------------------------------------
static void iisph_compute_velocity_changes(World& w) {
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        const Fluid& fi = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fi.n(); ++i) {
            float pi = w.pressures[f][i], rhoi = w.densities[f][i];
            V3 v = w.vc[f][i];
            for (const Contact& c : w.ff[f].lists[i]) {
                float mj = w.fluids[c.j_model].mass(c.j);
                float pj = w.pressures[c.j_model][c.j], rhoj = w.densities[c.j_model][c.j];
                v -= c.gradient * (w.dt * mj * (pi / (rhoi * rhoi) + pj / (rhoj * rhoj)));
            }
            for (const Contact& c : w.fb[f].lists[i]) {
                Boundary& b = w.boundaries[c.j_model];
                float mj = b.volumes[c.j] * fi.density0;
                V3 acc = c.gradient * (mj * pi / (rhoi * rhoi));
                v -= acc * w.dt;
                b.apply_force(c.j, acc * fi.mass(c.i));
            }
            w.vc[f][i] = v;
        }
    }
}
// ---- iisph_solver.rs:643-711 ----------------------------------------------------------------------
static bool iisph_step(World& w, V3 gravity) {
    bool ok = true;
    double t0 = now_ms();
    predict_advection(w, gravity);
    double t1 = now_ms();
    w.tm.nonpressure_ms += t1 - t0;
    timestep_advance(w);
    integrate_and_clear_accelerations(w);
    double t2 = now_ms();
    iisph_compute_dii(w);
    for (auto& v : w.pressures)
        for (float& p : v) p *= 0.5f;  // :673-677
    (void)compute_predicted_densities(w, &ok);
    iisph_compute_aii(w);
    // pressure_solve :422-456
    w.n_press_iter = w.n_press_eval = 0;
    uint32_t maxit = w.force_press >= 0 ? (uint32_t)w.force_press : w.max_pressure_iter;
    for (uint32_t i = 0; i < maxit; ++i) {
        iisph_compute_dij_pjl(w);
        float avg = iisph_compute_next_pressures(w);
        w.n_press_eval++;
        w.n_press_iter++;
        w.last_dens_err = avg;
        std::swap(w.pressures, w.next_pressures);
        if (w.force_press < 0 && avg <= w.max_density_error && i >= w.min_pressure_iter) break;
    }
    iisph_compute_velocity_changes(w);
    double t3 = now_ms();
    w.tm.pressure_ms += t3 - t2;
    // update_velocities_and_positions :406-420, zero vc :707-709
    for (size_t f = 0; f < w.fluids.size(); ++f) {
        Fluid& fl = w.fluids[f];
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)fl.n(); ++i) {
            fl.velocities[i] += w.vc[f][i];
            fl.positions[i] += fl.velocities[i] * w.dt;
            w.vc[f][i] = ZERO3;
        }
    }
    w.tm.integrate_ms += (t2 - t1) + (now_ms() - t3);
    return ok;
}

template <class T>
static void filter_from_mask(const std::vector<uint8_t>& mask, std::vector<T>& v) {  // helper.rs:4-12
    size_t k = 0;
    for (size_t i = 0; i < v.size(); ++i)
        if (!(i < mask.size() && mask[i])) v[k++] = v[i];
    v.resize(k);
}

// ---- dfsph_solver.rs:526-561 / iisph_solver.rs:479-537 + fluid.rs:88-98 -------------------------
static void init_with_fluids_and_removal(World& w) {
    size_t nf = w.fluids.size();
    for (auto* s : {&w.alphas, &w.densities, &w.predicted, &w.divergences, &w.aii, &w.pressures, &w.next_pressures})
        s->resize(nf);
    for (auto* s : {&w.vc, &w.dii, &w.dij_pjl}) s->resize(nf);
    for (size_t f = 0; f < nf; ++f) {
        Fluid& fl = w.fluids[f];
        size_t n = fl.n();
        for (auto* s : {&w.alphas, &w.densities, &w.predicted, &w.divergences, &w.aii, &w.pressures, &w.next_pressures})
            (*s)[f].resize(n, 0.f);
        for (auto* s : {&w.vc, &w.dii, &w.dij_pjl}) (*s)[f].resize(n, ZERO3);
        if (fl.num_deleted != 0) {
            for (auto* s : {&w.alphas, &w.densities, &w.predicted, &w.divergences, &w.aii, &w.pressures, &w.next_pressures})
                filter_from_mask(fl.deleted, (*s)[f]);
            for (auto* s : {&w.vc, &w.dii, &w.dij_pjl}) filter_from_mask(fl.deleted, (*s)[f]);
            filter_from_mask(fl.deleted, fl.positions);
            filter_from_mask(fl.deleted, fl.velocities);
            filter_from_mask(fl.deleted, fl.accelerations);
            filter_from_mask(fl.deleted, fl.volumes);
            fl.deleted.assign(fl.positions.size(), 0);
            fl.num_deleted = 0;
        }
    }
}

// ---- liquid_world.rs:67-158 -----------------------------------------------------------------------
static int world_step(World& w, float dt, V3 gravity) {
    double ts = now_ms();
    w.tm = Timings();
    w.total_step_size = dt;  // timestep_manager.rs:49-52 reset
    w.remaining_time = dt;
    init_with_fluids_and_removal(w);
    bool ok = true;
    while (!(w.remaining_time <= F32_EPS)) {  // is_done :56-58; runs exactly once
        double t0 = now_ms();
        insert_to_grid(w);
        double t1 = now_ms();
        compute_contacts(w);
        double t2 = now_ms();
        for (Boundary& b : w.boundaries)
            if (b.has_forces) std::fill(b.forces.begin(), b.forces.end(), ZERO3);  // coupling clears per substep
        evaluate_kernels(w);
        ok = compute_densities(w) && ok;
        double t3 = now_ms();
        w.tm.grid_ms += t1 - t0;
        w.tm.neighbors_ms += t2 - t1;
        w.tm.density_ms += t3 - t2;
        ok = (w.solver == 0 ? dfsph_step(w, gravity) : iisph_step(w, gravity)) && ok;
    }
    w.tm.step_ms = now_ms() - ts;
    if (!ok) {
        w.err = "zero density (reference assert dfsph_solver.rs:92,145,662)";
        return 5;
    }
    return 0;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
// C ABI of the oracle (prefix orc_; deliberately distinct from the product's sph_ symbols).
// ---------------------------------------------------------------------------------------------------
extern "C" {

struct orc_desc {
    int32_t solver;
    float particle_radius, smoothing_factor;
    uint32_t min_pressure_iter, max_pressure_iter;
    float max_density_error;
    uint32_t min_divergence_iter, max_divergence_iter;
    float max_divergence_error;
    float omega;
    int32_t sort_contacts;
    int32_t num_threads;
};

struct orc_stats {
    float step_ms, grid_ms, neighbors_ms, density_ms, divergence_ms, nonpressure_ms, pressure_ms, integrate_ms;
    uint32_t n_divergence_iter, n_pressure_iter, n_divergence_eval, n_pressure_eval;
    float last_divergence_error, last_density_error;
    uint64_t n_contacts;
    int32_t threads;
};

void* orc_world_create(const orc_desc* d) {
    World* w = new World();
    w->solver = d->solver;
    w->particle_radius = d->particle_radius;
    w->h = d->particle_radius * d->smoothing_factor * 2.0f;  // liquid_world.rs:44
    w->min_pressure_iter = d->min_pressure_iter;
    w->max_pressure_iter = d->max_pressure_iter;
    w->max_density_error = d->max_density_error;
    w->min_divergence_iter = d->min_divergence_iter;
    w->max_divergence_iter = d->max_divergence_iter;
    w->max_divergence_error = d->max_divergence_error;
    w->omega = d->omega;
    w->sort_contacts = d->sort_contacts;
#ifdef _OPENMP
    if (d->num_threads > 0) omp_set_num_threads(d->num_threads);
#endif
    return w;
}
void orc_world_destroy(void* p) { delete (World*)p; }
void orc_world_set_kernels(void* p, int kernel_density, int kernel_gradient) {
    ((World*)p)->kernel_density = kernel_density;
    ((World*)p)->kernel_gradient = kernel_gradient;
}
float orc_kernel_w_kind(int kind, float r, float h) { return w_scalar_kind(kind, r, h); }
float orc_kernel_dw_kind(int kind, float r, float h) { return dw_scalar_kind(kind, r, h); }

static void copy_v3(std::vector<V3>& dst, const float* src, size_t n) {
    dst.resize(n);
    if (src) std::memcpy(dst.data(), src, n * sizeof(V3));
    else std::fill(dst.begin(), dst.end(), ZERO3);
}

// Fluid::new fluid.rs:40-68
int orc_fluid_add(void* p, const float* pos, const float* vel, const float* volumes, size_t n, float density0,
                  uint32_t memberships, uint32_t filter) {
    World& w = *(World*)p;
    Fluid f;
    copy_v3(f.positions, pos, n);
    copy_v3(f.velocities, vel, n);
    f.accelerations.assign(n, ZERO3);
    float r = w.particle_radius;
    float pv = r * r * r * (float)(8.0 * 0.8);  // fluid.rs:117-118
    f.volumes.assign(n, pv);
    if (volumes) std::memcpy(f.volumes.data(), volumes, n * sizeof(float));
    f.density0 = density0;
    f.deleted.assign(n, 0);
    f.particle_radius = r;
    f.groups = {memberships, filter};
    w.fluids.push_back(std::move(f));
    return (int)w.fluids.size() - 1;
}
int orc_fluid_push_force(void* p, uint32_t fluid, int kind, const float* params) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size()) return 1;
    if (kind == F_WCSPH && params[1] != 0.f) return 1;  // see solve_wcsph
    Force f;
    f.kind = kind;
    std::memcpy(f.p, params, sizeof f.p);
    w.fluids[fluid].forces.push_back(std::move(f));
    return 0;
}
// LiquidWorld::particles_intersecting_aabb liquid_world.rs:211-243 over hgrid.rs:122-133 (cells key(mins)..=key(maxs) of the
// grid of the last step; distance of the CURRENT position to the box < particle_radius).  Output sorted by
// (kind, handle, index); returns the number found.
size_t orc_particles_in_aabb(void* p, const float* mins, const float* maxs, uint32_t* kinds, uint32_t* handles, uint32_t* indices, size_t cap) {
    World& w = *(World*)p;
    CellKey a = cell_key({mins[0], mins[1], mins[2]}, w.h), b = cell_key({maxs[0], maxs[1], maxs[2]}, w.h);
    struct Hit {
        uint32_t kind, handle, index;
        bool operator<(const Hit& o) const { return kind != o.kind ? kind < o.kind : handle != o.handle ? handle < o.handle : index < o.index; }
    };
    std::vector<Hit> hits;
    auto dist_ok = [&](V3 pt) {  // Aabb::distance_to_point(solid = true): norm of the per-axis excess
        float dx = std::max(std::max(mins[0] - pt.x, pt.x - maxs[0]), 0.f);
        float dy = std::max(std::max(mins[1] - pt.y, pt.y - maxs[1]), 0.f);
        float dz = std::max(std::max(mins[2] - pt.z, pt.z - maxs[2]), 0.f);
        return std::sqrt((dx * dx + dy * dy) + dz * dz) < w.particle_radius;
    };
    for (const auto& kv : w.grid) {
        const CellKey& k = kv.first;
        if (k.x < a.x || k.x > b.x || k.y < a.y || k.y > b.y || k.z < a.z || k.z > b.z) continue;
        for (const GridEntry& e : kv.second) {
            if (e.is_boundary) {
                if (e.model < w.boundaries.size() && e.particle < w.boundaries[e.model].n() && dist_ok(w.boundaries[e.model].positions[e.particle]))
                    hits.push_back({1u, e.model, e.particle});
            } else {
                if (e.model < w.fluids.size() && e.particle < w.fluids[e.model].n() && dist_ok(w.fluids[e.model].positions[e.particle]))
                    hits.push_back({0u, e.model, e.particle});
            }
        }
    }
    std::sort(hits.begin(), hits.end());
    for (size_t k = 0; k < hits.size() && k < cap; ++k) {
        kinds[k] = hits[k].kind;
        handles[k] = hits[k].handle;
        indices[k] = hits[k].index;
    }
    return hits.size();
}
int orc_fluid_push_host_force(void* p, uint32_t fluid, host_force_fn fn, void* user) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size() || !fn) return 1;
    Force f;
    f.kind = F_HOST;
    std::memset(f.p, 0, sizeof f.p);
    f.host_fn = fn;
    f.host_user = user;
    w.fluids[fluid].forces.push_back(std::move(f));
    return 0;
}
// Fluid::add_particles fluid.rs:126-150
int orc_fluid_append(void* p, uint32_t fluid, const float* pos, const float* vel, size_t n) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size()) return 1;
    w.edited = true;
    Fluid& f = w.fluids[fluid];
    float pv = f.particle_radius * f.particle_radius * f.particle_radius * (float)(8.0 * 0.8);
    for (size_t i = 0; i < n; ++i) {
        f.positions.push_back({pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]});
        f.velocities.push_back(vel ? V3{vel[3 * i], vel[3 * i + 1], vel[3 * i + 2]} : ZERO3);
        f.accelerations.push_back(ZERO3);
        f.volumes.push_back(pv);
        f.deleted.push_back(0);
    }
    return 0;
}
// Fluid::delete_particle_at_next_timestep fluid.rs:71-76
int orc_fluid_delete(void* p, uint32_t fluid, const uint8_t* mask, size_t n) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size() || n != w.fluids[fluid].n()) return 1;
    w.edited = true;
    Fluid& f = w.fluids[fluid];
    for (size_t i = 0; i < n; ++i)
        if (mask[i] && !f.deleted[i]) {
            f.deleted[i] = 1;
            f.num_deleted++;
        }
    return 0;
}
int orc_fluid_write(void* p, uint32_t fluid, const float* pos, const float* vel, size_t n) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size() || n != w.fluids[fluid].n()) return 1;
    if (pos) std::memcpy(w.fluids[fluid].positions.data(), pos, n * sizeof(V3));
    if (vel) std::memcpy(w.fluids[fluid].velocities.data(), vel, n * sizeof(V3));
    return 0;
}
size_t orc_fluid_count(void* p, uint32_t fluid) { return ((World*)p)->fluids[fluid].n(); }
int orc_fluid_read(void* p, uint32_t fluid, float* pos, float* vel) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size()) return 1;
    size_t n = w.fluids[fluid].n();
    if (pos) std::memcpy(pos, w.fluids[fluid].positions.data(), n * sizeof(V3));
    if (vel) std::memcpy(vel, w.fluids[fluid].velocities.data(), n * sizeof(V3));
    return 0;
}
// Boundary::new boundary.rs:28-46
int orc_boundary_add(void* p, const float* pos, const float* vel, size_t n, uint32_t memberships, uint32_t filter,
                     int want_forces) {
    World& w = *(World*)p;
    Boundary b;
    copy_v3(b.positions, pos, n);
    copy_v3(b.velocities, vel, n);
    b.volumes.assign(n, 0.f);
    b.has_forces = want_forces != 0;
    if (b.has_forces) {
        b.forces.assign(n, ZERO3);
        b.flocks = std::vector<SpinLock>(n);
    }
    b.groups = {memberships, filter};
    w.boundaries.push_back(std::move(b));
    return (int)w.boundaries.size() - 1;
}
int orc_boundary_write(void* p, uint32_t b, const float* pos, const float* vel, size_t n) {
    World& w = *(World*)p;
    if (b >= w.boundaries.size() || n != w.boundaries[b].n()) return 1;
    if (pos) std::memcpy(w.boundaries[b].positions.data(), pos, n * sizeof(V3));
    if (vel) std::memcpy(w.boundaries[b].velocities.data(), vel, n * sizeof(V3));
    return 0;
}
int orc_boundary_read(void* p, uint32_t b, float* volumes, float* forces) {
    World& w = *(World*)p;
    if (b >= w.boundaries.size()) return 1;
    Boundary& bd = w.boundaries[b];
    if (volumes) std::memcpy(volumes, bd.volumes.data(), bd.n() * sizeof(float));
    if (forces && bd.has_forces) std::memcpy(forces, bd.forces.data(), bd.n() * sizeof(V3));
    return 0;
}
int orc_world_step(void* p, float dt, const float* g) {
    World& w = *(World*)p;
    int rc = world_step(w, dt, {g[0], g[1], g[2]});
    if (rc == 0) w.edited = false;
    return rc;
}
void orc_world_force_iterations(void* p, int n_div, int n_press) {
    World& w = *(World*)p;
    w.force_div = n_div;
    w.force_press = n_press;
}
void orc_world_stats(void* p, orc_stats* s) {
    World& w = *(World*)p;
    s->step_ms = (float)w.tm.step_ms;
    s->grid_ms = (float)w.tm.grid_ms;
    s->neighbors_ms = (float)w.tm.neighbors_ms;
    s->density_ms = (float)w.tm.density_ms;
    s->divergence_ms = (float)w.tm.divergence_ms;
    s->nonpressure_ms = (float)w.tm.nonpressure_ms;
    s->pressure_ms = (float)w.tm.pressure_ms;
    s->integrate_ms = (float)w.tm.integrate_ms;
    s->n_divergence_iter = w.n_div_iter;
    s->n_pressure_iter = w.n_press_iter;
    s->n_divergence_eval = w.n_div_eval;
    s->n_pressure_eval = w.n_press_eval;
    s->last_divergence_error = w.last_div_err;
    s->last_density_error = w.last_dens_err;
    size_t nc = 0;
    for (auto& c : w.ff) nc += c.total();
    for (auto& c : w.fb) nc += c.total();
    for (auto& c : w.bb) nc += c.total();
    s->n_contacts = nc;
#ifdef _OPENMP
    s->threads = omp_get_max_threads();
#else
    s->threads = 1;
#endif
}
// what: same selectors as sph.h SPH_DBG_*
int orc_debug_read(void* p, uint32_t fluid, int what, float* out) {
    World& w = *(World*)p;
    if (fluid >= w.fluids.size()) return 1;
    size_t n = w.fluids[fluid].n();
    auto cpf = [&](const std::vector<std::vector<float>>& v) {
        if (fluid < v.size() && v[fluid].size() == n) std::memcpy(out, v[fluid].data(), n * sizeof(float));
        else std::memset(out, 0, n * sizeof(float));
    };
    auto cpv = [&](const std::vector<std::vector<V3>>& v) {
        if (fluid < v.size() && v[fluid].size() == n) std::memcpy(out, v[fluid].data(), n * sizeof(V3));
        else std::memset(out, 0, n * sizeof(V3));
    };
    switch (what) {
        case 0: cpf(w.densities); break;
        case 1: cpf(w.alphas); break;
        case 2: cpf(w.divergences); break;
        case 3: cpf(w.predicted); break;
        case 4: cpv(w.vc); break;
        case 5: for (size_t i = 0; i < n; ++i) out[i] = fluid < w.ff.size() && i < w.ff[fluid].lists.size() ? (float)w.ff[fluid].lists[i].size() : 0.f; break;
        case 6: for (size_t i = 0; i < n; ++i) out[i] = fluid < w.fb.size() && i < w.fb[fluid].lists.size() ? (float)w.fb[fluid].lists[i].size() : 0.f; break;
        case 7: cpf(w.pressures); break;
        case 8: cpv(w.dbg_acc); break;
        case 9: cpv(w.dii); break;
        case 10: cpf(w.aii); break;
        case 11: cpv(w.dij_pjl); break;
        case 12: case 13: case 14: case 15: case 16: case 17: case 18: case 19: {
            // plugin scratch of the fluid's last force of the kind; refused, as by the engine, unless that force has been
            // solved and no particle has been appended or deleted since (a write keeps the last solve's values)
            const int kind = what <= 13 ? F_HE2014 : what <= 15 ? F_DFSPH_VISC : F_BECKER;
            const Force* fc = nullptr;
            for (const Force& x : w.fluids[fluid].forces)
                if (x.kind == kind) fc = &x;
            if (!fc || w.edited) return 1;
            const size_t solved = kind == F_HE2014 ? fc->colors.size() : kind == F_DFSPH_VISC ? fc->betas.size() : fc->positions0.size();
            if (solved != n || (kind == F_DFSPH_VISC && fc->sr_target.size() != n)) return 1;
            for (size_t i = 0; i < n; ++i) switch (what) {
                case 12: out[i] = fc->colors[i]; break;
                case 13: out[i] = fc->gradcs[i]; break;
                case 14: std::memcpy(out + 36 * i, fc->betas[i].data(), 36 * sizeof(float)); break;
                case 15: std::memcpy(out + 6 * i, fc->sr_target[i].data(), 6 * sizeof(float)); break;
                case 16: out[i] = fc->volumes0[i]; break;
                case 17: std::memcpy(out + 9 * i, &fc->rotations[i].m[0][0], 9 * sizeof(float)); break;
                case 18: std::memcpy(out + 9 * i, &fc->grad_tr[i].m[0][0], 9 * sizeof(float)); break;
                default: std::memcpy(out + 6 * i, &fc->stress[6 * i], 6 * sizeof(float)); break;
            }
            break;
        }
        default: return 1;
    }
    return 0;
}
const char* orc_last_error(void* p) { return ((World*)p)->err.c_str(); }
float orc_kernel_w(float r, float h) { return w_scalar(r, h); }
float orc_kernel_dw(float r, float h) { return dw_scalar(r, h); }
float orc_cohesion_kernel(float r, float h) { return cohesion_kernel(r, h); }
float orc_adhesion_kernel(float r, float h) { return adhesion_kernel(r, h); }
int orc_max_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
}
