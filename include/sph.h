/*
 * sph.h — C ABI of the H100-native SPH fluid-step engine (libsalva_b200.so).
 *
 * This is the drop-in boundary for salva3d's solver path: every entry point
 * below is what a Rust `salva3d`-compatible shim binds over FFI in place of the
 * reference's in-process Rust implementation.  The reference interface each
 * entry point replaces is cited as  <file>:<line>  relative to the reference
 * tree (dimforge/salva @ 7eecdfb).
 *
 * Conventions
 *   - extern "C", no exceptions cross the boundary, no torch/CUDA types.
 *   - All pointers are caller-owned HOST memory, copied during the call; the
 *     library never retains them.  Vectors are tightly packed xyz f32 triples
 *     (the memory layout of Vec<Point3<f32>> / Vec<Vector3<f32>>).
 *   - A world has one logical owner (matches `&mut self`); calls on one world
 *     must be externally serialised; different worlds are independent.
 *     Callbacks (host forces, coupling managers) run on the calling thread
 *     inside sph_world_step*; they may call the read / write / query entry
 *     points of the SAME world re-entrantly, but not step it or add / remove
 *     fluids.
 *   - Fluid and boundary handles are (slot | generation << 16), like the
 *     reference's arena handles: removing an object invalidates only its own
 *     handle; a later add may reuse the slot under a new generation.
 *   - Errors: every call returns an sph_status; sph_last_error() gives text.
 *     Reference `assert!`/panic sites map to SPH_ERR_ZERO_DENSITY /
 *     SPH_ERR_INVALID; the Rust shim turns them back into panics.
 *   - There is NO CPU fallback: without a CUDA device sph_world_create fails
 *     with SPH_ERR_CUDA.
 */
#ifndef SALVA_B200_SPH_H
#define SALVA_B200_SPH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sph_world sph_world;

typedef enum {
    SPH_OK = 0,
    SPH_ERR_INVALID = 1,      /* bad argument / bad handle / reference assert (contacts.rs:165) */
    SPH_ERR_CUDA = 2,         /* CUDA runtime failure, or no device */
    SPH_ERR_OOM = 3,          /* device allocation failed / grid too large */
    SPH_ERR_NCCL = 4,         /* multi-GPU exchange failure */
    SPH_ERR_ZERO_DENSITY = 5  /* reference asserts dfsph_solver.rs:92,145,662 */
} sph_status;

/* Pressure solver selection: LiquidWorld::new(solver, ..) liquid_world.rs:39-57 */
enum { SPH_SOLVER_DFSPH = 0,  /* DFSPHSolver::new()  dfsph_solver.rs:54-70 */
       SPH_SOLVER_IISPH = 1   /* IISPHSolver::new()  iisph_solver.rs:48-64 */ };

/* Built-in NonPressureForce kinds (trait: solver/nonpressure_force.rs:10-30). */
enum { SPH_FORCE_XSPH_VISCOSITY = 0,        /* p[0]=fluid coeff, p[1]=boundary coeff   xsph_viscosity.rs:19-26 */
       SPH_FORCE_ARTIFICIAL_VISCOSITY = 1,  /* p[0]=fluid coeff, p[1]=boundary coeff, p[2]=alpha, p[3]=beta,
                                               p[4]=speed_of_sound                      artificial_viscosity.rs:27-38 */
       SPH_FORCE_AKINCI2013_TENSION = 2,    /* p[0]=tension coeff, p[1]=adhesion coeff akinci2013_surface_tension.rs:27-35 */
       SPH_FORCE_BECKER2009_ELASTICITY = 3, /* p[0]=young, p[1]=poisson, p[2]=nonlinear becker2009_elasticity.rs:60-76 */
       SPH_FORCE_HE2014_TENSION = 4,        /* p[0]=fluid tension coeff, p[1]=boundary tension coeff
                                               he2014_surface_tension.rs:21-29 */
       SPH_FORCE_WCSPH_TENSION = 5,         /* p[0]=fluid tension coeff, p[1]=boundary tension coeff (must be 0: the
                                               reference's boundary loop walks the FLUID contact list and indexes
                                               boundaries with it, wcsph_surface_tension.rs:66-83)
                                               wcsph_surface_tension.rs:21-27 */
       SPH_FORCE_DFSPH_VISCOSITY = 6,       /* p[0]=viscosity coeff in [0,1], p[1]=min_viscosity_iter (1),
                                               p[2]=max_viscosity_iter (50), p[3]=max_viscosity_error (0.01)
                                               dfsph_viscosity.rs:86-124 */
       SPH_FORCE_VORTICITY_CONFINEMENT = 7  /* p[0]=eps > 0 and finite, in m/s; p[1..7] unused.  No reference counterpart
                                               (Fedkiw, Stam & Jensen 2001; Macklin & Mueller 2013 section 6; DESIGN.md
                                               section 18).  For a particle i of the force's fluid f, with sums over i's
                                               fluid contacts j of fluid f (self included, contributing 0; boundaries
                                               contribute nothing and receive no reaction), V_j = m_j / rho_j of this
                                               step's densities and grad W_ij the solver's contact gradient at x_i - x_j,
                                               over the positions, velocities and densities the other forces read:
                                                 omega_i = sum_j V_j grad W_ij x (v_j - v_i)
                                                 eta_i   = sum_j V_j (|omega_j| - |omega_i|) grad W_ij
                                                 N_i     = eta_i / |eta_i| if |eta_i| > 0, else 0
                                                 a_i    += eps (N_i x omega_i)
                                               Refused (SPH_ERR_INVALID) for a NaN, infinite or non-positive eps and in
                                               slab-decomposed worlds. */ };

/* Kernel type parameters of the solver, DFSPHSolver<KernelDensity, KernelGradient> dfsph_solver.rs:17-20 /
 * IISPHSolver<..> iisph_solver.rs:17-20: contact.weight uses the density kernel, contact.gradient the gradient kernel
 * (helper.rs:24-25).  They are compile-time parameters in the reference and link-time ones here: libsalva_b200.so is
 * monomorphised on the cubic spline (sph_world_create rejects anything else), libsalva_b200_kernels.so — same source,
 * same ABI — serves every combination. */
enum { SPH_KERNEL_CUBIC_SPLINE = 0,  /* kernel/cubic_spline_kernel.rs:12-80 (default) */
       SPH_KERNEL_POLY6 = 1,         /* kernel/poly6_kernel.rs:12-40 */
       SPH_KERNEL_SPIKY = 2,         /* kernel/spiky_kernel.rs:12-40 */
       SPH_KERNEL_VISCOSITY = 3      /* kernel/viscosity_kernel.rs:12-51 */ };

typedef struct {
    int32_t  solver;                 /* SPH_SOLVER_* */
    float    particle_radius;        /* liquid_world.rs:41 */
    float    smoothing_factor;       /* h = r * sf * 2   liquid_world.rs:44 */
    uint32_t min_pressure_iter;      /* 1   dfsph_solver.rs:56 / iisph_solver.rs:50 */
    uint32_t max_pressure_iter;      /* 50 */
    float    max_density_error;      /* 0.05 */
    uint32_t min_divergence_iter;    /* 1   dfsph_solver.rs:59 (DFSPH only) */
    uint32_t max_divergence_iter;    /* 50 */
    float    max_divergence_error;   /* 0.1 */
    float    omega;                  /* 0.5  iisph_solver.rs:53 (IISPH only) */
    int32_t  device;                 /* CUDA device ordinal for this world (this rank's GPU) */
    int32_t  slab_rank;              /* multi-GPU slab decomposition along x: this world's slab index ... */
    int32_t  slab_count;             /* ... of slab_count slabs (1 = single GPU) */
    int32_t  deterministic;          /* 1: stable in-cell ordering => bit-reproducible run to run */
    int32_t  gather_backend;         /* must be 0; 1 (the tile backend) was removed. Kept so the struct layout does not
                                        change; sph_world_create refuses any other value with SPH_ERR_INVALID */
    int32_t  kernel_density;         /* SPH_KERNEL_*: KernelDensity  (0 = CubicSplineKernel) */
    int32_t  kernel_gradient;        /* SPH_KERNEL_*: KernelGradient (0 = CubicSplineKernel) */
} sph_world_desc;

typedef struct {
    int32_t kind;                    /* SPH_FORCE_* */
    float   p[8];
} sph_force_desc;

/* Per-step statistics; supersedes the reference's wall-clock Counters
 * (counters/mod.rs:17-30) with CUDA-event timings, and exposes the iteration
 * counts the reference only has as commented println! (dfsph_solver.rs:449-452). */
typedef struct {
    float    step_ms;                /* counters.step_time */
    float    grid_ms;                /* cd.grid_insertion_time: cell hash + counting sort + reorder */
    float    neighbors_ms;           /* cd.neighborhood_search_time: neighbour-list build */
    float    density_ms;             /* evaluate_kernels + compute_densities + compute_alphas */
    float    divergence_ms;          /* divergence_solve */
    float    nonpressure_ms;         /* solver.non_pressure_resolution_time */
    float    pressure_ms;            /* pressure_solve (the roofline-capture region) */
    float    integrate_ms;
    float    divergence_eval_ms;     /* sum over compute_divergences launches              (kernel K4a) */
    float    divergence_update_ms;   /* sum over compute_velocity_changes_for_divergence   (kernel K4b) */
    float    predict_density_ms;     /* sum over compute_predicted_densities launches      (kernel K8a) */
    float    pressure_update_ms;     /* sum over compute_velocity_changes launches         (kernel K8b) */
    uint32_t n_divergence_iter;      /* velocity-change updates executed in divergence_solve */
    uint32_t n_pressure_iter;        /* velocity-change updates executed in pressure_solve */
    uint32_t n_divergence_eval;      /* compute_divergences launches */
    uint32_t n_pressure_eval;        /* compute_predicted_densities / compute_next_pressures launches */
    float    last_divergence_error;
    float    last_density_error;
    uint64_t n_fluid_particles;
    uint64_t n_boundary_particles;
    uint64_t n_contacts;             /* cd.ncontacts: ff + fb + bb */
    uint32_t max_neighbors;          /* widest fluid neighbour list this step */
    uint32_t grid_dims[3];
    uint64_t kernel_launches;        /* CUDA kernels launched by this step */
    uint32_t n_ghost_particles;      /* multi-GPU: ghost particles received from the neighbour slabs this step */
    uint32_t n_migrated;             /* multi-GPU: particles handed over to / received from neighbour slabs */
    uint32_t n_exchanges;            /* multi-GPU: ghost-refresh exchanges (ncclSend/Recv groups) this step */
    uint32_t n_substeps;             /* counters.nsubsteps (liquid_world.rs:86): substeps the step ran, 0 when no solver ran.
                                        Over a substepped step the times, iteration / evaluation counts and kernel_launches are
                                        sums, max_neighbors the maximum, everything else the last substep's */
} sph_step_stats;

/* sph_debug_read() selectors: solver scratch in ORIGINAL particle order. */
enum { SPH_DBG_DENSITY = 0,            /* densities            dfsph_solver.rs:41  */
       SPH_DBG_ALPHA = 1,              /* alphas               dfsph_solver.rs:40  */
       SPH_DBG_DIVERGENCE = 2,         /* divergences          dfsph_solver.rs:43  */
       SPH_DBG_PREDICTED_DENSITY = 3,  /* predicted_densities  dfsph_solver.rs:42  */
       SPH_DBG_VELOCITY_CHANGE = 4,    /* velocity_changes (3 floats/particle) dfsph_solver.rs:44 */
       SPH_DBG_NUM_FLUID_CONTACTS = 5, /* len(ff list) as float, self included contacts.rs:83-87 */
       SPH_DBG_NUM_BOUNDARY_CONTACTS = 6,
       SPH_DBG_PRESSURE = 7,           /* IISPH pressures      iisph_solver.rs:37 (after a host edit: the carried ones) */
       SPH_DBG_ACCELERATION = 8,       /* fluid.accelerations (3 floats/particle), after forces, before integrate */
       /* IISPH scratch (SPH_ERR_INVALID for DFSPH, and before the first IISPH step) */
       SPH_DBG_IISPH_DII = 9,          /* dii (3 floats/particle)                      iisph_solver.rs:32 */
       SPH_DBG_IISPH_AII = 10,         /* aii                                          iisph_solver.rs:33 */
       SPH_DBG_IISPH_DIJ_PJL = 11,     /* dij_pjl of the last pressure iteration (3)   iisph_solver.rs:34 */
       /* Plugin scratch of the fluid's last force of the kind (SPH_ERR_INVALID unless that force has been solved since
        * particles were last added or deleted; after sph_fluid_write it holds the last solve's values).  `out` holds width * cap floats, width as noted (1 if not). */
       SPH_DBG_HE2014_COLOR = 12,      /* He2014 colours                               he2014_surface_tension.rs:16 */
       SPH_DBG_HE2014_GRADC = 13,      /* He2014 squared colour-gradient norms         he2014_surface_tension.rs:17 */
       SPH_DBG_VISC_BETA = 14,         /* DFSPHViscosity beta (36, row-major 6x6)      dfsph_viscosity.rs:99 */
       SPH_DBG_VISC_TARGET = 15,       /* DFSPHViscosity strain-rate target (6)        dfsph_viscosity.rs:100 */
       SPH_DBG_EL_VOLUME0 = 16,        /* Becker2009 rest volumes                      becker2009_elasticity.rs:48-58 */
       SPH_DBG_EL_ROTATION = 17,       /* Becker2009 rotation (9, row-major)           becker2009_elasticity.rs:48-58 */
       SPH_DBG_EL_GRAD_TR = 18,        /* Becker2009 deformation_gradient_tr (9, row-major) becker2009_elasticity.rs:48-58 */
       SPH_DBG_EL_STRESS = 19,         /* Becker2009 stress (6: x y z w a b)           becker2009_elasticity.rs:48-58 */
       /* The last sph_world_update_diffuse's values per fluid particle (SPH_ERR_INVALID unless that update selected the
        * fluid with its current particle count; 0 for particles with non-finite positions) */
       SPH_DBG_DIFFUSE_NORMAL = 20,    /* n = -grad phi / |grad phi| (3)                DESIGN.md section 16 */
       SPH_DBG_DIFFUSE_TRAPPED_AIR = 21, /* I_ta before clamping */
       SPH_DBG_DIFFUSE_WAVE_CREST = 22,  /* I_wc before clamping (0 where v^ . n < 0.6) */
       SPH_DBG_DIFFUSE_KINETIC = 23,     /* E_k before clamping */
       SPH_DBG_DIFFUSE_COUNT = 24,       /* n_d, the particles it asked to emit, as float */
       SPH_DBG_FLUID_LIST_BITS = 25,     /* the width in bits (16 or 32) of the fluid list entries the last neighbour search
                                          * stored, the same for every particle (DESIGN.md section 4a.18) */
       /* Plugin scratch of the fluid's last SPH_FORCE_VORTICITY_CONFINEMENT, under the rule of selectors 12-19 */
       SPH_DBG_VORTICITY = 26,           /* omega (3) */
       SPH_DBG_VORTICITY_ETA = 27        /* eta (3), the unnormalised gradient of |omega| */ };

/* LiquidWorld::new  liquid_world.rs:39-57 */
void       sph_world_desc_default(sph_world_desc* desc);
sph_status sph_world_create(const sph_world_desc* desc, sph_world** out);
void       sph_world_destroy(sph_world* w);

/* LiquidWorld::add_fluid liquid_world.rs:161 + Fluid::new fluid.rs:40-68.
 * volumes == NULL -> 0.8*(2r)^3 (fluid.rs:110-120); vel == NULL -> zeros. */
sph_status sph_fluid_add(sph_world* w, const float* pos_xyz, const float* vel_xyz, const float* volumes,
                         size_t n, float density0, uint32_t memberships, uint32_t filter, uint32_t* handle);
/* fluid.nonpressure_forces.push(..)  fluid.rs:14; forces run in push order (dfsph_solver.rs:590). */
sph_status sph_fluid_push_force(sph_world* w, uint32_t fluid, const sph_force_desc* force);
/* User-defined NonPressureForce plugins (trait solver/nonpressure_force.rs:10-30; e.g. examples3d/custom_forces3.rs:66-90):
 * arbitrary HOST code that adds to fluid.accelerations.  At the force's slot in push order the library hands the
 * callback the fluid's particles in ORIGINAL index order (host copies) and takes the accelerations back.  `dt` / `inv_dt`
 * are the TimestepManager values the reference passes at that point (the previous step's: dfsph_solver.rs:693-702).
 * Like the reference's predict_advection (dfsph_solver.rs:580-603, iisph_solver.rs alike), every step that runs the solver
 * (the world holds at least one fluid particle) calls each force once, that of an empty fluid too, with n == 0 (its
 * pointers may then be NULL).  Contact lists are not materialised for these callbacks: see sph_fluid_push_host_force2. */
typedef void (*sph_host_force_fn)(void* user, float dt, float inv_dt, float kernel_radius, size_t n, const float* positions_xyz,
                                  const float* velocities_xyz, const float* densities, float* accelerations_xyz);
sph_status sph_fluid_push_host_force(sph_world* w, uint32_t fluid, sph_host_force_fn fn, void* user);

/* The same plugin hook with the COMPLETE argument list of NonPressureForce::solve (nonpressure_force.rs:15-27):
 * timestep, kernel radius, fluid_fluid_contacts, fluid_boundaries_contacts, the fluid, the boundaries, the densities.
 * Contacts (contacts.rs:12-27 `Contact {i_model, j_model, i, j, weight, gradient}`) are materialised on request as CSR
 * over the fluid's particles in ORIGINAL index order: the contacts of particle i are entries ff_offsets[i] ..
 * ff_offsets[i+1]; `j` is the neighbour's index INSIDE its own fluid / boundary, `j_model` that object's slot
 * (handle & 0xFFFF; == ctx.fluid_index for same-fluid contacts); the self contact (j == i, gradient 0) is included, as
 * in the reference.  An empty fluid's force is called too, with n == 0 and ff_offsets == fb_offsets == {0}.  All
 * pointers are host memory owned by the library for the duration of the call. */
enum { SPH_HOST_FORCE_CONTACTS = 1u,    /* fill ff_* / fb_* */
       SPH_HOST_FORCE_BOUNDARIES = 2u   /* fill boundaries[] (positions, velocities, volumes) */ };
typedef struct {
    size_t n;
    const float* positions_xyz;   /* boundary.positions  boundary.rs:13 */
    const float* velocities_xyz;  /* boundary.velocities boundary.rs:15 */
    const float* volumes;         /* boundary.volumes    boundary.rs:17 (this step's) */
} sph_boundary_view;
typedef struct {
    float dt, inv_dt;             /* TimestepManager::dt() / inv_dt() at the call (the previous step's: dfsph_solver.rs:693-702) */
    float kernel_radius, particle_radius;
    uint32_t fluid;               /* handle of the fluid the force belongs to */
    uint32_t fluid_index;         /* its slot == the i_model / j_model value of same-fluid contacts */
    float density0;
    size_t n;                     /* particles of the fluid */
    const float* positions_xyz;
    const float* velocities_xyz;
    const float* densities;       /* solve()'s `densities` argument */
    const float* volumes;         /* fluid.volumes (NULL in slab-decomposed worlds) */
    float* accelerations_xyz;     /* fluid.accelerations: add to it in place */
    const uint32_t* ff_offsets;   /* n + 1 */
    const uint32_t* ff_j;
    const uint32_t* ff_j_model;
    const float* ff_weight;       /* contact.weight   = W(|x_ij|)      helper.rs:19 */
    const float* ff_gradient_xyz; /* contact.gradient = grad W(x_ij)   helper.rs:24-25 */
    const uint32_t* fb_offsets;
    const uint32_t* fb_j;
    const uint32_t* fb_j_model;
    const float* fb_weight;
    const float* fb_gradient_xyz;
    size_t n_boundaries;          /* number of boundary slots (removed ones have n == 0) */
    const sph_boundary_view* boundaries;
} sph_host_force_ctx;
typedef void (*sph_host_force_fn2)(void* user, const sph_host_force_ctx* ctx);
sph_status sph_fluid_push_host_force2(sph_world* w, uint32_t fluid, sph_host_force_fn2 fn, void* user, uint32_t flags);
/* Fluid::add_particles fluid.rs:126-150.  The new particles go to the end of the fluid's index range with the default volume,
 * zero velocity_changes and zero IISPH pressure.  Their ids count up from 1 + the largest id among the fluid's current
 * particles (those marked for deletion included; 0 for an empty fluid), so an id is never held by two live particles of a
 * fluid, and a fluid nothing was deleted from keeps the ids 0..n-1.  SPH_ERR_INVALID (nothing appended) when the new ids
 * would pass 0xFFFFFFFF, which only ids given through sph_fluid_set_ids / sph_fluid_replace_particles can bring about.  In a
 * slab-decomposed world the largest id is taken over this rank's particles only: give appended particles world-wide ids
 * with sph_fluid_set_ids there. */
sph_status sph_fluid_append(sph_world* w, uint32_t fluid, const float* pos_xyz, const float* vel_xyz, size_t n);
/* Fluid::delete_particle_at_next_timestep fluid.rs:71-76; applied at the next step (fluid.rs:88-98). */
sph_status sph_fluid_delete(sph_world* w, uint32_t fluid, const uint8_t* mask, size_t n);
/* Host-side edits between steps through fluids_mut() (liquid_world.rs:186-188). NULL = leave unchanged. */
sph_status sph_fluid_write(sph_world* w, uint32_t fluid, const float* pos_xyz, const float* vel_xyz, size_t n);
/* Reads fluid.positions / fluid.velocities in ORIGINAL index order. NULL = skip. */
sph_status sph_fluid_read(sph_world* w, uint32_t fluid, float* pos_xyz, float* vel_xyz, size_t cap, size_t* n);
sph_status sph_fluid_count(sph_world* w, uint32_t fluid, size_t* n);
/* LiquidWorld::remove_fluid liquid_world.rs:171-173 (the handle dies, the others stay valid). */
sph_status sph_fluid_remove(sph_world* w, uint32_t fluid);
/* Replaces a fluid's whole particle set: positions, velocities, velocity_changes (dfsph_solver.rs:44, the part of the
 * velocity DFSPH carries between steps; NULL = zeros) and ids (NULL = 0..n-1).  Used by the slab worlds' plane re-balancing
 * (salva_b200/slab.py rebalance), where particles change rank wholesale.  sph_debug_read(SPH_DBG_VELOCITY_CHANGE) reads vc. */
sph_status sph_fluid_replace_particles(sph_world* w, uint32_t fluid, const float* pos_xyz, const float* vel_xyz, const float* vc_xyz,
                                       const uint32_t* ids, size_t n);
/* Zero-copy read-back for renderers (testbed_plugin.rs:361-376 copies fluid.positions every frame): DEVICE pointers to
 * packed xyz f32 in ORIGINAL index order, valid until the next call on this world. */
sph_status sph_fluid_map_positions(sph_world* w, uint32_t fluid, const float** device_xyz, size_t* n);
sph_status sph_fluid_map_velocities(sph_world* w, uint32_t fluid, const float** device_xyz, size_t* n);

/* LiquidWorld::add_boundary liquid_world.rs:166 + Boundary::new boundary.rs:28-46.
 * want_forces != 0  <=>  boundary.forces = Some(..) (boundary.rs:21). */
sph_status sph_boundary_add(sph_world* w, const float* pos_xyz, const float* vel_xyz, size_t n,
                            uint32_t memberships, uint32_t filter, int want_forces, uint32_t* handle);
/* CouplingManager::update_boundaries rewriting boundary particles (coupling_manager.rs:12-20). */
sph_status sph_boundary_write(sph_world* w, uint32_t boundary, const float* pos_xyz, const float* vel_xyz, size_t n);
/* LiquidWorld::remove_boundary liquid_world.rs:176-178. */
sph_status sph_boundary_remove(sph_world* w, uint32_t boundary);
/* A coupled collider re-samples its boundary every step with a varying particle count (fluids_pipeline.rs:175-245:
 * positions.clear(); push(..)): replaces the whole particle set. */
sph_status sph_boundary_set_particles(sph_world* w, uint32_t boundary, const float* pos_xyz, const float* vel_xyz, size_t n);
sph_status sph_boundary_count(sph_world* w, uint32_t boundary, size_t* n);
/* boundary.forces read by CouplingManager::transmit_forces (coupling_manager.rs:22-27). */
sph_status sph_boundary_read_forces(sph_world* w, uint32_t boundary, float* f_xyz, size_t cap);
/* boundary.volumes after compute_boundary_volumes (dfsph_solver.rs:72-96). */
sph_status sph_boundary_read_volumes(sph_world* w, uint32_t boundary, float* volumes, size_t cap);

/* LiquidWorld::particles_intersecting_aabb  liquid_world.rs:211-243: the particles of the cells [key(mins), key(maxs)]
 * of the grid built by the LAST step (hgrid.rs:122-133) whose CURRENT position is closer than particle_radius to the
 * box.  Entry k is (kinds[k] = 0 fluid / 1 boundary, handles[k], indices[k] = index inside that object), sorted by
 * (kind, handle, index) — the reference's order is hash-map order.  *n = number found (may exceed cap; only cap
 * entries are written).  Empty before the first step, like the reference's empty grid.  SPH_ERR_INVALID while host
 * edits (write/append/delete) are pending: the cell grid of the last step no longer describes those particles. */
sph_status sph_world_particles_in_aabb(sph_world* w, const float mins[3], const float maxs[3], uint32_t* kinds, uint32_t* handles,
                                       uint32_t* indices, size_t cap, size_t* n);

/* LiquidWorld::particles_intersecting_shape liquid_world.rs:246-281 for the shapes a C ABI can name (parry `Shape` trait
 * objects cannot cross it): the cells of the posed shape's AABB (shape.compute_aabb(pos)), every particle in them with
 * shape.distance_to_point(pos, p, solid = true) <= particle_radius.  rotation_rowmajor == NULL: identity.  Output as
 * sph_world_particles_in_aabb. */
enum { SPH_SHAPE_BALL = 1,     /* p[0] = radius */
       SPH_SHAPE_CUBOID = 2,   /* p[0..2] = half extents */
       SPH_SHAPE_CAPSULE = 3   /* p[0] = half height (segment along local y), p[1] = radius */ };
/* parry Cylinder / Cone, axis along local y, p[0] = half height a, p[1] = (base) radius r, both finite and >= 0 (zero gives a
 * disc, a segment, a flat or a needle cone).  The cylinder is sqrt(x^2 + z^2) <= r, |y| <= a; the cone's apex is (0, a, 0)
 * and its base disc lies at y = -a: |y| <= a, sqrt(x^2 + z^2) <= r (a - y) / (2a).  Local AABB [-r, -a, -r]-[r, a, r]; the
 * posed AABB is parry's tight support-map box, not centred on the translation for the cone.  Projection, inside test and
 * tie order: DESIGN.md section 10.  Kinds 5 and 6 are accepted by sph_world_particles_in_shape, sph_collider_register and
 * sph_world_sample_shape. */
enum { SPH_SHAPE_CYLINDER = 5, SPH_SHAPE_CONE = 6 };
typedef struct {
    int32_t kind;
    float   p[4];
} sph_shape;
sph_status sph_world_particles_in_shape(sph_world* w, const sph_shape* shape, const float translation[3], const float rotation_rowmajor[9],
                                        uint32_t* kinds, uint32_t* handles, uint32_t* indices, size_t cap, size_t* n);

/* salva3d::sampling::shape_surface_ray_sample / shape_volume_ray_sample  sampling/ray_sampling.rs:9-24 (the 3-D branch of
 * :27-231) on the device.  The shape is in its local frame.  SPH_SHAPE_HEIGHTFIELD is parry's HeightField: rows of the
 * height matrix run along z and columns along x, x and z span [-0.5, 0.5] * scale, heights are multiplied by scale[1], and
 * cell (row i, column j) is split along its (x0, z1)-(x1, z0) diagonal; its triangles are hit from both sides.
 * sph_world_particles_in_shape and sph_collider_register refuse it (they have no sph_heightfield argument): a heightfield
 * goes to sph_world_particles_in_heightfield and sph_collider_register_heightfield.  The world supplies the device, the
 * stream and the scratch memory; the world's particles are not touched.  Output: *n points (packed xyz) in ascending
 * order of their quantised (x, y, z) keys, where the reference's order is HashSet order; *n may exceed cap, only cap points are
 * written.  SPH_ERR_INVALID (nothing written) for a particle_radius that is not finite and positive, a shape parameter
 * that is negative or not finite, a heightfield with nrows or ncols below 2, a non-finite height or a scale component that
 * is not finite and positive, and when a quantised coordinate reaches 2^21 (or an axis needs more than 2^21 rays).
 * SPH_ERR_OOM when the candidate buffers cannot be allocated.  See DESIGN.md section 11. */
enum { SPH_SHAPE_HEIGHTFIELD = 4 };  /* sph_shape.p unused; the field is the sph_heightfield argument */
enum { SPH_SAMPLE_SURFACE = 0, SPH_SAMPLE_VOLUME = 1 };
typedef struct {
    uint32_t     nrows, ncols;
    const float* heights;  /* nrows * ncols, row-major */
    float        scale[3];
} sph_heightfield;
sph_status sph_world_sample_shape(sph_world* w, int32_t method, const sph_shape* shape, const sph_heightfield* heightfield,
                                  float particle_radius, float* xyz, size_t cap, size_t* n);
/* LiquidWorld::particles_intersecting_shape liquid_world.rs:246-281 for a parry HeightField: the cells of compute_aabb(pos)
 * (the field's local AABB is not centred: centre R c + t, half extents |R| e), every particle in them with
 * shape.distance_to_point(pos, p, solid = true) <= particle_radius, where parry's heightfield point query has is_inside always
 * false: the distance is the unsigned distance to the closest point of the triangulated surface.  Heightfield checks as
 * sph_world_sample_shape (SPH_ERR_INVALID, nothing written); output and pending-edit rules as sph_world_particles_in_shape.
 * See DESIGN.md section 10. */
sph_status sph_world_particles_in_heightfield(sph_world* w, const sph_heightfield* heightfield, const float translation[3],
                                              const float rotation_rowmajor[9], uint32_t* kinds, uint32_t* handles, uint32_t* indices,
                                              size_t cap, size_t* n);

/* LiquidWorld::step  liquid_world.rs:62-158 */
sph_status sph_world_step(sph_world* w, float dt, const float gravity[3]);

/* n_steps calls of sph_world_step(w, dt, gravity) in one call (LiquidWorld::step liquid_world.rs:62-158, repeated).  Step 1
 * runs as sph_world_step does; steps 2..n_steps run as one CUDA graph whose Jacobi loops end on the device, with no host round
 * trip between steps.  The results equal those of the n_steps calls, bit for bit in deterministic mode.  *steps_done is the
 * number of steps that returned SPH_OK; on an error the failing step is applied as sph_world_step applies it, and its status
 * is returned.  sph_world_stats afterwards merges the steps as substeps are merged: times and counts summed, max_neighbors the
 * widest, the rest the last step's, n_substeps the steps run, kernel_launches the host's launches (a graph launch counts
 * one), phase times 0 for steps run in the graph, step_ms the device time of the call, and grid_dims, when the last step ran in
 * the graph, the dims of the graph's grid (the fluid and boundary AABB with 4 cells to spare on every side, DESIGN.md
 * section 13) rather than of the grid that step would have had on its own.  A driver older than CUDA 12.4 runs every step as
 * sph_world_step does (records with on_device 0).  DFSPH on one GPU only: SPH_ERR_INVALID,
 * nothing changed, for IISPH, Becker2009 or DFSPHViscosity forces, host forces, registered colliders, substepping on
 * (cfl_coeff != 0) and slab-decomposed worlds.  n_steps == 0 does nothing.  See DESIGN.md section 13. */
sph_status sph_world_step_many(sph_world* w, float dt, const float gravity[3], uint32_t n_steps, uint32_t* steps_done);

/* What one step did (sph_step_stats' per-step counts; liquid_world.rs:84-148 counters) */
typedef struct {
    uint32_t n_divergence_iter, n_pressure_iter, n_divergence_eval, n_pressure_eval;
    float    last_divergence_error, last_density_error;
    uint32_t max_neighbors;
    uint32_t on_device;            /* 1: this step ran inside the graph, 0: on the per-step path */
    uint64_t n_contacts;
} sph_step_record;
/* One record per step of the last sph_world_step / sph_world_step_many call, in order: min(cap, *n) are written, and *n
 * (which may exceed cap) is the count. */
sph_status sph_world_read_step_records(sph_world* w, sph_step_record* out, size_t cap, size_t* n);

/* trait CouplingManager (coupling/coupling_manager.rs:9-28) + LiquidWorld::step_with_coupling (liquid_world.rs:67-158).
 * update_boundaries runs after this substep's FLUID particles are in the cell grid and before the boundaries are
 * (liquid_world.rs:86-103): particle queries issued from it return fluid particles only, and it may rewrite boundaries
 * (sph_boundary_write / sph_boundary_set_particles) and push fluid particles out (sph_fluid_read / sph_fluid_write), as
 * DynamicContactSampling does (fluids_pipeline.rs:192-255).  transmit_forces runs after the solve (liquid_world.rs:146)
 * and reads sph_boundary_read_forces.  dt / inv_dt are the TimestepManager's values at each call. */
typedef struct {
    void (*update_boundaries)(void* user, sph_world* w, float dt, float inv_dt, float h, float particle_radius);
    void (*transmit_forces)(void* user, sph_world* w, float dt, float inv_dt);
    void* user;
} sph_coupling_manager;
sph_status sph_world_step_with_coupling(sph_world* w, float dt, const float gravity[3], const sph_coupling_manager* coupling);

/* Collider coupling on the device: the rapier integration's ColliderCouplingSet / ColliderCouplingManager
 * (integrations/rapier/fluids_pipeline.rs:72-287) run inside sph_world_step, where update_boundaries runs
 * (liquid_world.rs:86-103).  The rigid-body engine stays with the caller: before each step it hands over each collider's
 * pose and body velocities (sph_collider_set_state), after it reads the impulse the fluid applied (sph_collider_read_impulse).
 * Colliders cannot be combined with a host sph_coupling_manager in one step, nor used in slab-decomposed worlds; a collider
 * whose boundary was removed is inert and no longer counts. */
enum { SPH_SAMPLING_STATIC = 0,    /* ColliderSampling::StaticSampling(points)  fluids_pipeline.rs:69,180-191 */
       SPH_SAMPLING_CONTACT = 1 }; /* ColliderSampling::DynamicContactSampling  fluids_pipeline.rs:71,192-255: every step, after the
   fluids are in the cell grid, each fluid particle in the cells of the posed shape's AABB loosened by 1.5 h whose predicted
   position p = pos + vel * dt (the lagging dt) lies in that AABB is projected onto the shape's surface; a particle inside is
   pushed out along the projection normal by depth + 0.1 particle_radius and loses its velocity into the shape; the projection
   becomes a boundary particle with the body's velocity at that WORLD point, unless p lies more than 1.5 h outside.  Colliders
   run in slot order; the boundary holds its samples ordered by the sampled particle's fluid slot, then index.  A ball's
   centre yields no sample; a point on a capsule's, cylinder's or cone's axis projects along local +x.  A heightfield (parry's point query has
   is_inside always false, point_heightfield.rs) never pushes: it only samples its closest surface points.  See DESIGN.md
   section 10. */
enum { SPH_BODY_NONE = 0,     /* collider.parent() == None: velocity 0, boundary.forces left as it is (fluids_pipeline.rs:163-171),
                                 no impulse (transmit_forces needs the parent body, :273-276) */
       SPH_BODY_FIXED = 1,    /* !body.is_dynamic(): boundary.forces = None, no impulse */
       SPH_BODY_DYNAMIC = 2 };/* boundary.forces = Some, cleared every step */
typedef struct {
    float   translation[3];        /* collider.position(): world = rotation * local + translation */
    float   rotation_rowmajor[9];
    int32_t body;                  /* SPH_BODY_* */
    float   linvel[3], angvel[3], world_com[3];  /* RigidBody::velocity_at_point(p) = linvel + angvel x (p - world_com) */
} sph_collider_state;
/* ColliderCouplingSet::register_coupling(boundary, collider, sampling)  fluids_pipeline.rs:98-114.  StaticSampling: the n_points
 * local points (packed xyz) become the boundary's particles; every step they are posed by the collider's state, with the
 * velocity velocity_at_point(pt) evaluated at the LOCAL point pt, as fluids_pipeline.rs:183 does (a quirk of the reference,
 * reproduced).  `shape` may be NULL for StaticSampling.  SPH_SAMPLING_CONTACT needs a ball, cuboid, capsule, cylinder or cone `shape` with
 * finite, non-negative parameters and n_points == 0; the boundary keeps its particles until the next step refills it, and its
 * particle count changes every step (sph_boundary_count).  The engine owns the boundary's particle set from then on:
 * sph_boundary_write / _set_particles refuse it.  A boundary can be coupled to one collider at a time.  The initial state
 * is the identity pose with SPH_BODY_NONE.  Handles are slot | generation << 16. */
sph_status sph_collider_register(sph_world* w, uint32_t boundary, int32_t sampling, const sph_shape* shape, const float* local_points_xyz,
                                 size_t n_points, uint32_t* collider);
/* register_coupling(boundary, collider, ColliderSampling::DynamicContactSampling) fluids_pipeline.rs:98-114, 192-255 for a
 * collider whose shape is a parry HeightField (StaticSampling needs no shape: use sph_collider_register).  The heights are
 * copied into device memory owned by the collider, so the caller's buffer may be freed; sph_collider_unregister and
 * sph_world_destroy free it.  The heightfield never pushes fluid (is_inside is always false in parry's heightfield point
 * query): each candidate's closest surface point becomes a sample unless it lies more than 1.5 h away.  All other rules of
 * sph_collider_register apply.  Heightfield checks as sph_world_sample_shape (SPH_ERR_INVALID, nothing written);
 * SPH_ERR_OOM when the heights cannot be allocated. */
sph_status sph_collider_register_heightfield(sph_world* w, uint32_t boundary, const sph_heightfield* heightfield, uint32_t* collider);
/* The collider's pose and body for the next steps (the reference reads collider.position() and the parent body each
 * update_boundaries, fluids_pipeline.rs:159-186).  A StaticSampling collider whose state is bit-equal to the one of its
 * last step leaves its boundary unchanged, so the boundary's sort and volumes are reused as for a static boundary. */
sph_status sph_collider_set_state(sph_world* w, uint32_t collider, const sph_collider_state* state);
/* ColliderCouplingManager::transmit_forces fluids_pipeline.rs:263-287 of the last step: linear = sum of force * dt,
 * angular = sum of (p - world_com) x force * dt over the boundary's particles, with the step's dt.  Zero when the body is
 * not SPH_BODY_DYNAMIC, when the boundary is empty or was removed, and before the first step. */
sph_status sph_collider_read_impulse(sph_world* w, uint32_t collider, float linear[3], float angular[3]);
/* ColliderCouplingSet::unregister_coupling fluids_pipeline.rs:119-122: the boundary stays, with its last particle set. */
sph_status sph_collider_unregister(sph_world* w, uint32_t collider);
/* Particle sinks and sources of a fluid, applied on the device at the start of every step (DESIGN.md section 14).  They do on
 * the device what faucet3.rs:69-105 does from a host callback before each step: mark the particles below a plane with
 * delete_particle_at_next_timestep (fluid.rs:100-104) and append a sheet with add_particles (fluid.rs:126-150) every 0.06 s.
 * Each sph_world_step / sph_world_step_with_coupling call that gets past its refusals counts as one step, a step of
 * dt <= FLT_EPSILON included.  In it, after the marks of sph_fluid_delete are applied (liquid_world.rs:79-81) and before the
 * boundaries, colliders, grid and solver:
 *   1. every particle that a sink of its fluid removes, tested at its position at the start of the step, is deleted; the
 *      survivors keep their order (fluid.rs:88-98);
 *   2. every source that fires appends its template to the end of its fluid's index range, in registration order, exactly
 *      as sph_fluid_append would: default volume, zero velocity_changes and IISPH pressure.  The ids count up from 1 + the
 *      largest id the fluid held at the start of the step, marked and sunk particles included, continuing from one source
 *      to the next.
 * The result equals reading the positions, sph_fluid_delete with the sinks' mask and sph_fluid_append of each firing template
 * before the step, bit for bit in deterministic mode, without a round trip of the particles through the host.  Up to 64 sinks
 * and 64 sources per world; handles are slot | generation << 16.  sph_fluid_remove removes its fluid's sinks and sources.
 * Snapshots store neither, and sph_world_snapshot_load leaves them and their step counts as they are.  Slab-decomposed worlds
 * refuse them (SPH_ERR_INVALID), and sph_world_step_many refuses to run while any is registered.  A step whose emissions
 * would number ids past 2^32 - 1 is refused with SPH_ERR_INVALID before it changes anything. */
typedef struct {
    float   lo[3], hi[3];  /* a particle is in the box iff lo[a] <= x[a] < hi[a] on every axis (f32 comparisons; +-INFINITY allowed) */
    int32_t outside;       /* 0: removes the particles in the box (faucet3.rs:77-81: y < -2 is lo = -inf, hi = (inf, -2, inf));
                              1: removes every particle not in the box (a domain sink; non-finite positions are in no box) */
} sph_sink_desc;
/* A sink of `fluid` (faucet3.rs:74-86).  SPH_ERR_INVALID, nothing changed, for a NaN bound, lo > hi on an axis or outside
 * other than 0 / 1. */
sph_status sph_fluid_add_sink(sph_world* w, uint32_t fluid, const sph_sink_desc* sink, uint32_t* sink_handle);
sph_status sph_sink_remove(sph_world* w, uint32_t sink);
/* A source of `fluid` (faucet3.rs:88-103): the n particles of pos_xyz (packed xyz) with velocities vel_xyz (NULL: zero) are
 * copied to the device now and appended on the first step after this call and on every interval-th step after it (interval
 * counts steps: faucet3's 0.06 s at dt = 1 / 200 is 12).  SPH_ERR_INVALID, nothing changed, for n == 0, a NULL template or
 * interval == 0. */
sph_status sph_fluid_add_source(sph_world* w, uint32_t fluid, const float* pos_xyz, const float* vel_xyz, size_t n, uint32_t interval,
                                uint32_t* source_handle);
sph_status sph_source_remove(sph_world* w, uint32_t source);
/* How many particles of `fluid` the sinks removed and the sources emitted in the last step (0 before any step).  NULL = skip. */
sph_status sph_fluid_read_step_edits(sph_world* w, uint32_t fluid, uint32_t* removed, uint32_t* emitted);

/* Fluid surface meshes on the device (DESIGN.md section 15).  The field phi(x) = sum_j V_j W(|x - x_j|) sums over the particles
 * of the selected fluids (boundaries are not included), with V_j the particle's volume, W the world's density kernel and h, and
 * the positions of the last step (before the first step: those given).  Inside settled fluid phi ~ rho / rho0 ~ 1.  It is
 * sampled on the lattice p_ijk = origin + spacing * (i, j, k), x fastest, with origin[a] = spacing * floor(lo[a] / spacing)
 * and n[a] = ceil((hi[a] - origin[a]) / spacing) + 1 points per axis (f32 operations; a coordinate is origin[a] + (float)i *
 * spacing, a product and then a sum), so the lattices of successive frames and of different boxes share their points.  A point
 * is inside iff phi >= iso.  Every lattice cube is split into the 6 tetrahedra (0, e_a, e_a + e_b, 1) and each is polygonised
 * by a 16-case table, so the mesh is watertight and no case is ambiguous.  Vertices: one per crossed lattice edge, at
 * x = p_a + t (p_b - p_a) with t = (iso - phi_a) / (phi_b - phi_a), a the inside end; ordered by the point owning the edge
 * (x fastest), then by its direction +x, +y, +z, +x+y, +x+z, +y+z, +x+y+z.  Triangles: ordered by cube, tetrahedron
 * (permutations xyz, xzy, yxz, yzx, zxy, zyx) and table order; counter-clockwise seen from outside (the side of lower phi).
 * Normals (optional): -grad phi / |grad phi| at the vertex with the world's gradient kernel, 0 where the gradient is 0.  In
 * deterministic mode field and mesh are bit-identical run to run and do not depend on the fluids' slot order.
 * The default box (lo[0] > hi[0]) is the selected fluids' AABB grown by h on every side: phi is 0 on its border and every
 * surface closes.  A caller box clips the lattice, and surfaces are open where the box cuts them. */
typedef struct {
    float   iso;           /* finite, > 0 */
    float   spacing;       /* finite, > 0 */
    float   lo[3], hi[3];  /* box to mesh; lo[0] > hi[0] = the selected fluids' AABB grown by h */
    int32_t normals;       /* 1: also compute vertex normals (a second gather), 0: skip */
} sph_surface_desc;
/* Extracts the surface of fluids[0..n_fluids) (n_fluids == 0: every fluid).  The field and mesh stay in device buffers of the
 * world until the next extraction or sph_world_destroy; the step, its grid and its cached graphs are not touched.  No fluid
 * particles give 0 vertices and 0 triangles.  SPH_ERR_INVALID, nothing changed and the previous mesh kept, for NaN or
 * out-of-range desc fields, lo > hi on some axes but not all, a non-finite caller box, stale or duplicate fluid handles,
 * slab-decomposed worlds, calls from inside a coupling or host-force callback, and pending host edits (sph_fluid_write /
 * _append / _delete after the last step: step first).  SPH_ERR_OOM, nothing changed, when the lattice would exceed 2^31
 * points, the vertex or triangle count would pass 2^32 - 1, or an allocation fails. */
sph_status sph_world_extract_surface(sph_world* w, const uint32_t* fluids, size_t n_fluids, const sph_surface_desc* desc,
                                     size_t* n_vertices, size_t* n_triangles);
/* The last extraction's mesh: packed xyz vertices, their normals (NULL = skip) and 3 vertex indices per triangle.
 * SPH_ERR_INVALID when vcap or tcap is below the counts, or normals_xyz is not NULL and the extraction ran with normals = 0. */
sph_status sph_world_read_surface(sph_world* w, float* vertices_xyz, float* normals_xyz, size_t vcap, uint32_t* triangles, size_t tcap);
/* Device pointers to the same arrays (d_normals_xyz NULL when not computed), valid until the next extraction: the zero-copy
 * path for renderers, like sph_fluid_map_positions.  Any output pointer may be NULL. */
sph_status sph_world_map_surface(sph_world* w, const float** d_vertices_xyz, const float** d_normals_xyz, const uint32_t** d_triangles);
/* phi on the last extraction's lattice, x fastest, with its origin and point counts (0 before any extraction and when no
 * lattice was built).  phi == NULL: only origin and dims are written.  SPH_ERR_INVALID when cap is below the point count. */
sph_status sph_world_read_surface_field(sph_world* w, float* phi, size_t cap, float origin[3], uint32_t dims[3]);

/* Anisotropic fluid surfaces (Yu & Turk 2013, "Reconstructing surfaces of particle-based fluids using anisotropic kernels";
 * DESIGN.md section 17).  The same lattice, inside rule, polygonisation, orderings and sph_world_read_surface_field as
 * sph_world_extract_surface; only phi and the normals differ.  Over the selected fluids' particles with finite positions x_i
 * (the positions of the last step; before the first step: those given), with volumes V_i, the world's h and its kernels:
 *   1. Neighbours of i: the j != i with |x_ij|^2 <= h^2 under the step's unfused float32 pair test (the test of
 *      sph_world_update_diffuse step 3); N_i their count.  Weights w_ij = 1 - (|x_ij| / h)^3; i itself enters the sums below
 *      with w_ii = 1 but is not counted in N_i.
 *   2. Weighted mean x^w_i = sum w_ij x_j / sum w_ij; centre x_bar_i = (1 - lambda) x_i + lambda x^w_i.
 *   3. Covariance C_i = sum w_ij (x_j - x^w_i)(x_j - x^w_i)^T / sum w_ij, eigenvalues s1 >= s2 >= s3 >= 0, orthonormal
 *      eigenvectors e1, e2, e3 (cyclic Jacobi in float32, at most 8 sweeps).
 *   4. Radii: if N_i >= N_eps and s1 > 0, a_k = h max(s_k, s1 / k_r) / s1, so a1 = h and every a_k lies in [h / k_r, h];
 *      otherwise a1 = a2 = a3 = k_n h with the axes x, y, z.
 *   5. Kernel: G_i = sum_k e_k e_k^T / a_k, W_i(x) = (h^3 / (a1 a2 a3)) W(h |G_i (x - x_bar_i)|) with W the world's density
 *      kernel.  W_i integrates to 1 and vanishes outside the ellipsoid of semi-axes a_k <= h around x_bar_i.
 *   6. Field phi(x) = sum_i V_i W_i(x); normals -grad phi / |grad phi| with grad W_i(x) = (h^3 / (a1 a2 a3)) h G_i grad W(u),
 *      u = h G_i (x - x_bar_i), the world's gradient kernel, grad W(u) = 0 for |u|^2 <= eps^2, and 0 where grad phi = 0.
 * Two deliberate departures from the paper: (a) the neighbourhood radius is h, not 2h, so the ellipsoid pass is the same
 * 27-cell gather as every other pass; (b) the paper's global scale k_s is replaced by per-particle normalisation, the longest
 * semi-axis being exactly h: every ellipsoid then lies inside the sphere of radius h around its centre, so the field pass
 * keeps the 27-cell gather around the centre's cell, where a global k_s could stretch an axis past h and silently lose
 * contributions.  With lambda = 0, k_r = 1 and k_n = 1 every kernel is the isotropic one and phi is section 15's phi (in
 * exact arithmetic).  Radii: a_k = h max(s_k / s1, 1 / k_r) in float32, the ratio first.  Defaults
 * (sph_surface_anisotropy_default): lambda = 0.9, k_r = 1, k_n = 1, N_eps = 6, project values, not the paper's: smoothed
 * centres with round kernels.  That is the setting found to mesh a jittered slab flatter than sph_world_extract_surface
 * without inner shells (DESIGN.md section 17).  k_r > 1 stretches the kernels along the surface, but with the longest axis
 * held at h their volume shrinks, so in jittered fluid the field can dip below iso under the surface layer and the mesh gains
 * closed inner shells; DESIGN.md section 17 has the measurements.  Every centre lies in the convex hull of the positions,
 * so the default box still closes every surface.  Ellipsoids are computed for every selected particle: a caller box clips
 * only the lattice, so a small box over a large fluid pays for the whole fluid's ellipsoids.  In deterministic mode field,
 * mesh and ellipsoids are bit-identical run to run and do not depend on the fluids' slot order. */
typedef struct {
    float    smoothing;        /* lambda in [0, 1] */
    float    max_ratio;        /* k_r in [1, 1000] (every semi-axis >= h / 1000) */
    float    isolated_radius;  /* k_n in [0.001, 1], in units of h */
    uint32_t min_neighbours;   /* N_eps */
} sph_surface_anisotropy;
void sph_surface_anisotropy_default(sph_surface_anisotropy* a);
/* sph_world_extract_surface with the anisotropic field.  SPH_ERR_INVALID, nothing changed and the previous mesh, field and
 * ellipsoids kept, for everything sph_world_extract_surface refuses and for NaN or out-of-range anisotropy fields.  Besides
 * its SPH_ERR_OOM cases, SPH_ERR_OOM when the selected fluids' AABB spans more than 2^31 cells of width h (the ellipsoid pass
 * bins every particle, where the isotropic field bins only those the lattice reaches). */
sph_status sph_world_extract_surface_anisotropic(sph_world* w, const uint32_t* fluids, size_t n_fluids, const sph_surface_desc* desc,
                                                 const sph_surface_anisotropy* aniso, size_t* n_vertices, size_t* n_triangles);
/* The last extraction's ellipsoids of one fluid, in that fluid's particle order (sph_fluid_read's): the centre x_bar and
 * 12 floats per particle, (e1, a1, e2, a2, e3, a3), with a1 >= a2 >= a3.  n = 0 after an isotropic extraction or when the
 * fluid was not selected.  A non-finite position gives its position as the centre and zero axes.  centres_xyz and axes
 * NULL: only n is written; SPH_ERR_INVALID when cap is below n. */
sph_status sph_world_read_surface_ellipsoids(sph_world* w, uint32_t fluid, float* centres_xyz, float* axes, size_t cap, size_t* n);
/* Device pointers to the same rows (NULL when n = 0), valid until the next extraction: the zero-copy input of a splatting
 * renderer.  Either output pointer may be NULL. */
sph_status sph_world_map_surface_ellipsoids(sph_world* w, uint32_t fluid, const float** d_centres_xyz, const float** d_axes, size_t* n);

/* Diffuse particles on the device: spray, foam and air bubbles (Ihmsen et al. 2012; DESIGN.md section 16).  A one-way
 * post-process: sph_world_update_diffuse reads the selected fluids at the positions and velocities of the last step (before
 * the first step: those given) and never writes the fluid.  The step, its grid and its cached graphs are not touched.  One
 * update, in order:
 *   1. The selected fluids' particles are binned into cells of width h (in (fluid slot, id) order within a cell in
 *      deterministic mode); particles with non-finite positions are left out.
 *   2. n_i = -grad phi(x_i) / |grad phi(x_i)|, phi = sum_j V_j W over the selected fluids within h (the surface extractor's
 *      field, the world's gradient kernel); 0 where grad phi = 0.
 *   3. Over the j with |x_ij|^2 <= h^2 (the step's unfused float32 pair test), x_ij = x_i - x_j, v_ij = v_i - v_j,
 *      W~(r) = 1 - r / h:  I_ta = sum |v_ij| (1 - v^_ij . x^_ij) W~ (terms with |x_ij| = 0 or |v_ij| = 0 are 0);
 *      kappa = sum over j with x_ij . n_i > 0 of (1 - n_i . n_j) W~, I_wc = kappa if |v_i| > 0 and v_i . n_i / |v_i| >= 0.6,
 *      else 0;  E_k = 0.5 V_i rho0 |v_i|^2.  Each is clamped as Phi(I, lo, hi) = (min(I, hi) - min(I, lo)) / (hi - lo), and
 *      n_d = floor(Phi_k (k_ta Phi_ta + k_wc Phi_wc) dt + u), each operation rounded once in float32 in this order (products,
 *      then the sum, then * Phi_k, * dt, + u), min(a, b) = b < a ? b : a, NaN counting 0.  u = hash(seed, counter, slot, id,
 *      0, stream 0) mapped to (h >> 8) 2^-24 (salva_b200/csrc/sph_hash.h), so small dt still emits on average.
 *   4. In binned order, fluid particle i emits particles k = 0 .. n_d - 1, appended behind the survivors of the last update;
 *      those past `capacity` are dropped.  With X_r, X_theta, X_h the hash's streams 1, 2, 3 for k, r = r_p sqrt(X_r),
 *      theta = 2 pi X_theta and e1, e2 Duff et al. 2017's orthonormal basis around v^_f:  o = r cos theta e1 + r sin theta e2,
 *      x = x_f + o + X_h dt v_f, v = v_f + o, life = lifetime.
 *   5. Every diffuse particle, old and new: n_n = the fluid particles within h, v~ = sum v_j W / sum W (the density
 *      kernel; 0 when the sum is 0).  Spray (n_n < spray_below): v += dt g, x += dt v.  Bubble (n_n > bubble_above):
 *      v += -dt k_b g + k_d (v~ - v), x += dt v.  Foam (otherwise): v = v~, x += dt v~, life -= dt; only foam ages.
 *   6. Foam with life <= 0 and every particle outside lo <= x < hi (non-finite positions included) are removed; the
 *      survivors keep their order.  The update counter increments.
 * In deterministic mode the set is bit-identical run to run and does not depend on the fluids' slot order.  The defaults
 * (sph_diffuse_desc_default) are tuning values for scenes of particle radius about 0.05, not values from the paper. */
enum { SPH_DIFFUSE_SPRAY = 0, SPH_DIFFUSE_FOAM = 1, SPH_DIFFUSE_BUBBLE = 2 };
typedef struct {
    float    ta_min, ta_max;      /* trapped-air clamp, finite, ta_min < ta_max */
    float    wc_min, wc_max;      /* wave-crest clamp */
    float    k_min, k_max;        /* kinetic-energy clamp */
    float    k_ta, k_wc;          /* emission rates per second, finite, >= 0 */
    float    lifetime;            /* foam lifetime, finite, > 0 */
    float    k_b;                 /* bubble buoyancy, finite, >= 0 */
    float    k_d;                 /* bubble drag towards the fluid, in [0, 1] */
    uint32_t spray_below;         /* spray: fewer fluid neighbours than this */
    uint32_t bubble_above;        /* bubble: more fluid neighbours than this; spray_below <= bubble_above + 1 */
    uint32_t capacity;            /* most diffuse particles kept, > 0 */
    uint32_t seed;
    float    lo[3], hi[3];        /* particles outside lo <= x < hi are removed; lo <= hi, no NaN (infinities allowed) */
} sph_diffuse_desc;
typedef struct {
    uint64_t emitted;             /* appended by this update */
    uint64_t dropped;             /* asked for past capacity */
    uint64_t expired;             /* foam whose life ran out */
    uint64_t left_box;            /* removed outside the box (non-finite positions included) */
    uint64_t spray, foam, bubble; /* the set after the update, by kind */
} sph_diffuse_stats;
void sph_diffuse_desc_default(sph_diffuse_desc* d);
/* Advances the world's diffuse set by one frame of length dt under gravity, from fluids[0..n_fluids) (n_fluids == 0: every
 * fluid).  stats may be NULL.  SPH_ERR_INVALID, nothing changed, for NaN or out-of-range desc fields, ta/wc/k min >= max,
 * dt not finite and > 0, a non-finite gravity, lo > hi on any axis, capacity 0, stale or duplicate fluid handles,
 * slab-decomposed worlds, calls from inside a coupling or host-force callback, and pending host edits.  SPH_ERR_OOM,
 * nothing changed, past 2^31 binning cells or when an allocation fails.  A set larger than capacity (capacity lowered
 * between updates) emits nothing and is not truncated. */
sph_status sph_world_update_diffuse(sph_world* w, const uint32_t* fluids, size_t n_fluids, const sph_diffuse_desc* desc, float dt,
                                    const float gravity[3], sph_diffuse_stats* stats);
/* The set in order: packed xyz positions and velocities, kinds (SPH_DIFFUSE_*) and lives; NULL = skip; *n = count.
 * SPH_ERR_INVALID when cap is below the count and some output is not NULL. */
sph_status sph_world_read_diffuse(sph_world* w, float* pos_xyz, float* vel_xyz, uint8_t* kind, float* life, size_t cap, size_t* n);
/* Device pointers to the same arrays, valid until the next update or clear: the zero-copy path for renderers.  Any output
 * pointer may be NULL. */
sph_status sph_world_map_diffuse(sph_world* w, const float** d_pos_xyz, const float** d_vel_xyz, const uint8_t** d_kind,
                                 const float** d_life, size_t* n);
/* Empties the set; the update counter keeps counting.  Snapshots do not store the set, and sph_world_snapshot_load leaves
 * it as it is. */
sph_status sph_world_clear_diffuse(sph_world* w);

/* boundary.positions / velocities (boundary.rs:13-15) in ORIGINAL index order.  NULL = skip; *n = particle count. */
sph_status sph_boundary_read(sph_world* w, uint32_t boundary, float* pos_xyz, float* vel_xyz, size_t cap, size_t* n);

/* Snapshot / restore of everything the solver carries ACROSS steps: positions, velocities, velocity_changes
 * (dfsph_solver.rs:44, carried :704-706), the lagging dt / inv_dt (timestep_manager.rs:29-30), IISPH warm-start pressures
 * (iisph_solver.rs:673-677), Becker-2009 rest pose and rotations (becker2009_elasticity.rs:84-135), volumes, particle ids,
 * slab planes.  The blob restores into a world with the same fluids / forces / boundaries pushed in the same order (the
 * scene description stays with the caller).  In deterministic mode a restored run is bit-identical to the original. */
sph_status sph_world_snapshot_size(sph_world* w, size_t* bytes);
sph_status sph_world_snapshot_save(sph_world* w, void* buffer, size_t capacity, size_t* written);
sph_status sph_world_snapshot_load(sph_world* w, const void* buffer, size_t length);
/* Parity/bench aid: run exactly this many velocity-change updates in the next steps'
 * divergence / pressure loops instead of the error-driven break (negative = free running). */
sph_status sph_world_force_iterations(sph_world* w, int32_t n_divergence, int32_t n_pressure);
/* CFL-bounded substeps: the TimestepManager's cfl_coeff / min_num_substeps / max_num_substeps (timestep_manager.rs:21-46),
 * whose rule the reference leaves commented out (compute_substep :87-94 returns the whole step).  cfl_coeff == 0 (the
 * default) turns substepping off: every step is one substep, as in the reference.  Otherwise a step of length T runs
 * substeps k = 0, 1, ... while the remaining time R_k > FLT_EPSILON (R_0 = T).  Each computes, after the non-pressure forces,
 * m = max over the fluid particles of |v + a * R_k|^2 and d = (2 r) / sqrt(m) * cfl_coeff (+inf when m == 0), and runs
 * n_k = clamp(ceil(R_k / d), max(1, min_substeps - k), max(1, max_substeps - k)) even parts of R_k: dt_k = R_k / n_k,
 * R_{k+1} = R_k - dt_k.  So dt_k <= d unless max_substeps binds, the substeps add up to T (f32 rounding aside), and their
 * count lies in [min_substeps, max_substeps].  SPH_ERR_INVALID, nothing changed, for a NaN or negative cfl_coeff (+inf is
 * allowed), min_substeps == 0, min_substeps > max_substeps, and in a slab-decomposed world (slab_count > 1).  Snapshots
 * do not carry these settings.  See DESIGN.md section 12. */
sph_status sph_world_set_substepping(sph_world* w, float cfl_coeff, uint32_t min_substeps, uint32_t max_substeps);
/* The lengths dt_k of the last step's substeps in order (counters.nsubsteps of them, liquid_world.rs:86): min(cap, *n)
 * are written, and *n (which may exceed cap) is the count; 0 when the step ran no solver. */
sph_status sph_world_read_substeps(sph_world* w, float* dts, size_t cap, size_t* n);
sph_status sph_world_stats(sph_world* w, sph_step_stats* out);
/* LiquidWorld::h / particle_radius  liquid_world.rs:201-208 */
float      sph_world_h(const sph_world* w);
float      sph_world_particle_radius(const sph_world* w);
sph_status sph_debug_read(sph_world* w, uint32_t fluid, int what, float* out, size_t cap);
const char* sph_last_error(const sph_world* w);
const char* sph_version(void);

/* Caller-visible particle ids (default: the index a particle had when it was added with sph_fluid_add; for appended
 * particles see sph_fluid_append).  They follow particles when the sort reorders them, through deletions, and when a particle
 * migrates to another rank's slab.  The ids of a fluid are the in-cell sort key: they must be unique within the fluid for
 * a run to be bit-reproducible from a snapshot, which the library's own ids are and ids given here should be. */
sph_status sph_fluid_set_ids(sph_world* w, uint32_t fluid, const uint32_t* ids, size_t n);
sph_status sph_fluid_read_ids(sph_world* w, uint32_t fluid, uint32_t* ids, size_t cap);

/* Multi-GPU (one process per GPU; the reference has no counterpart: SURVEY.md §8e).  1-D slab decomposition along x:
 * the world of rank r owns the particles whose cell column floor(x / h) lies in [cell_lo, cell_hi) (INT32_MIN / INT32_MAX
 * = open end), the host adds only those to it (plus ALL boundary particles), and every step the library exchanges
 * one-cell ghost columns with ranks r-1 / r+1 (ncclSend/ncclRecv over NVLink) and migrates particles that crossed a
 * plane.  In a slab world the index order of a fluid (sph_fluid_read / _write / _delete) is the engine's sorted order of the moment
 * and changes with every step: track particles by id (sph_fluid_set_ids / sph_fluid_read_ids), which migration preserves.
 * Either hand over an initialised ncclComm_t (attach) or let the library create one from a unique id that
 * rank 0 obtained with sph_nccl_unique_id() and the host's own plumbing (torch.distributed) broadcast. */
sph_status sph_nccl_unique_id(char out_id[128]);
sph_status sph_world_create_nccl(sph_world* w, const char unique_id[128], int rank, int nranks);
sph_status sph_world_attach_nccl(sph_world* w, void* nccl_comm, int rank, int nranks);
sph_status sph_world_set_slab(sph_world* w, int32_t cell_lo, int32_t cell_hi);

#ifdef __cplusplus
}
#endif
#endif /* SALVA_B200_SPH_H */
