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
       SPH_FORCE_DFSPH_VISCOSITY = 6        /* p[0]=viscosity coeff in [0,1], p[1]=min_viscosity_iter (1),
                                               p[2]=max_viscosity_iter (50), p[3]=max_viscosity_error (0.01)
                                               dfsph_viscosity.rs:86-124 */ };

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
    int32_t  gather_backend;         /* 0: L1/texture gathers over 32-bit global lists (default, fastest measured);
                                        1: tile-staged shared memory via TMA bulk copies + 16-bit tile-local lists */
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
    uint32_t reserved_;
} sph_step_stats;

/* sph_debug_read() selectors: solver scratch in ORIGINAL particle order. */
enum { SPH_DBG_DENSITY = 0,            /* densities            dfsph_solver.rs:41  */
       SPH_DBG_ALPHA = 1,              /* alphas               dfsph_solver.rs:40  */
       SPH_DBG_DIVERGENCE = 2,         /* divergences          dfsph_solver.rs:43  */
       SPH_DBG_PREDICTED_DENSITY = 3,  /* predicted_densities  dfsph_solver.rs:42  */
       SPH_DBG_VELOCITY_CHANGE = 4,    /* velocity_changes (3 floats/particle) dfsph_solver.rs:44 */
       SPH_DBG_NUM_FLUID_CONTACTS = 5, /* len(ff list) as float, self included contacts.rs:83-87 */
       SPH_DBG_NUM_BOUNDARY_CONTACTS = 6,
       SPH_DBG_PRESSURE = 7,           /* IISPH pressures      iisph_solver.rs:37  */
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
       SPH_DBG_EL_STRESS = 19          /* Becker2009 stress (6: x y z w a b)           becker2009_elasticity.rs:48-58 */ };

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
 * Contact lists are not materialised for callbacks (pass-through of ParticlesContacts is a later row). */
typedef void (*sph_host_force_fn)(void* user, float dt, float inv_dt, float kernel_radius, size_t n, const float* positions_xyz,
                                  const float* velocities_xyz, const float* densities, float* accelerations_xyz);
sph_status sph_fluid_push_host_force(sph_world* w, uint32_t fluid, sph_host_force_fn fn, void* user);

/* The same plugin hook with the COMPLETE argument list of NonPressureForce::solve (nonpressure_force.rs:15-27):
 * timestep, kernel radius, fluid_fluid_contacts, fluid_boundaries_contacts, the fluid, the boundaries, the densities.
 * Contacts (contacts.rs:12-27 `Contact {i_model, j_model, i, j, weight, gradient}`) are materialised on request as CSR
 * over the fluid's particles in ORIGINAL index order: the contacts of particle i are entries ff_offsets[i] ..
 * ff_offsets[i+1]; `j` is the neighbour's index INSIDE its own fluid / boundary, `j_model` that object's slot
 * (handle & 0xFFFF; == ctx.fluid_index for same-fluid contacts); the self contact (j == i, gradient 0) is included, as
 * in the reference.  All pointers are host memory owned by the library for the duration of the call. */
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
/* Fluid::add_particles fluid.rs:126-150 */
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
typedef struct {
    int32_t kind;
    float   p[4];
} sph_shape;
sph_status sph_world_particles_in_shape(sph_world* w, const sph_shape* shape, const float translation[3], const float rotation_rowmajor[9],
                                        uint32_t* kinds, uint32_t* handles, uint32_t* indices, size_t cap, size_t* n);

/* LiquidWorld::step  liquid_world.rs:62-158 */
sph_status sph_world_step(sph_world* w, float dt, const float gravity[3]);

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
   centre yields no sample; a point on a capsule's axis projects along local +x.  See DESIGN.md section 10. */
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
 * reproduced).  `shape` may be NULL for StaticSampling.  SPH_SAMPLING_CONTACT needs a ball, cuboid or capsule `shape` with
 * finite, non-negative parameters and n_points == 0; the boundary keeps its particles until the next step refills it, and its
 * particle count changes every step (sph_boundary_count).  The engine owns the boundary's particle set from then on:
 * sph_boundary_write / _set_particles refuse it.  A boundary can be coupled to one collider at a time.  The initial state
 * is the identity pose with SPH_BODY_NONE.  Handles are slot | generation << 16. */
sph_status sph_collider_register(sph_world* w, uint32_t boundary, int32_t sampling, const sph_shape* shape, const float* local_points_xyz,
                                 size_t n_points, uint32_t* collider);
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
sph_status sph_world_stats(sph_world* w, sph_step_stats* out);
/* LiquidWorld::h / particle_radius  liquid_world.rs:201-208 */
float      sph_world_h(const sph_world* w);
float      sph_world_particle_radius(const sph_world* w);
sph_status sph_debug_read(sph_world* w, uint32_t fluid, int what, float* out, size_t cap);
const char* sph_last_error(const sph_world* w);
const char* sph_version(void);

/* Caller-visible particle ids (default: the index a particle had when it was added).  They follow particles when the
 * sort reorders them and when a particle migrates to another rank's slab. */
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
