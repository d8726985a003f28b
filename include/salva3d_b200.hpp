// salva3d_b200.hpp — header-only C++ host mirror of salva3d's solver-path API on top of the C ABI (include/sph.h).
//
// The reference's host language (Rust) is not part of this build, so the host side above the C ABI is
// provided in C++ with the reference's type names, constructor arguments and error behaviour (reference panics /
// assert! sites become exceptions).  Mirrors (paths under the reference's src/):
//   LiquidWorld::{new, add_fluid, add_boundary, step, fluids, boundaries, h, particle_radius}  liquid_world.rs:39-208
//   Fluid::{new, add_particles, delete_particle_at_next_timestep, num_particles, particle_mass}  object/fluid.rs:40-196
//   Boundary::new                                                                              object/boundary.rs:28-46
//   InteractionGroups::{default, test}                                                         object/interaction_groups.rs:64-79
//   DFSPHSolver::new / IISPHSolver::new (public tunables)       solver/pressure/dfsph_solver.rs:54-70, iisph_solver.rs:48-64
//   XSPHViscosity / ArtificialViscosity / Akinci2013SurfaceTension / Becker2009Elasticity ::new  solver/{viscosity,surface_tension,elasticity}/*.rs
//   DFSPHSolver<KernelDensity, KernelGradient> with CubicSpline / Poly6 / Spiky / Viscosity kernels        dfsph_solver.rs:17-20, kernel/*.rs
//   LiquidWorld::{remove_fluid, remove_boundary, step_with_coupling, particles_intersecting_shape}          liquid_world.rs:67-178,246-281
//   trait CouplingManager                                                                                    coupling/coupling_manager.rs:9-28
//   NonPressureForce::solve with contacts and boundaries (CustomNonPressureForceWithContacts)                nonpressure_force.rs:15-27
//   ColliderCouplingSet::{register_coupling, unregister_coupling} + ColliderSampling::{StaticSampling, DynamicContactSampling},
//   run on the device
//   (the rigid bodies stay with the caller: set_collider_state before a step, collider_impulse after it)   fluids_pipeline.rs:64-287
// Every call goes to libsalva_b200.so (CUDA); there is no CPU path.
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "sph.h"

namespace salva3d {

using Real = float;  // lib.rs:199
struct Vector3 {
    Real x = 0, y = 0, z = 0;
};
using Point3 = Vector3;  // tightly packed xyz f32 triples == Vec<Point3<f32>> memory layout

struct InteractionGroups {  // interaction_groups.rs:20-79
    uint32_t memberships = 1u, filter = 0xFFFFFFFFu;
    bool test(const InteractionGroups& rhs) const { return (memberships & rhs.filter) != 0 && (rhs.memberships & filter) != 0; }
};

struct NonPressureForce {  // solver/nonpressure_force.rs:10-30 (built-in forces carry a descriptor the engine executes)
    virtual ~NonPressureForce() {}
    virtual sph_force_desc descriptor() const = 0;
};
// User-defined force: arbitrary host code, as a `dyn NonPressureForce` is in the reference (examples3d/custom_forces3.rs:66-90).
struct CustomNonPressureForce : NonPressureForce {
    virtual void solve(Real dt, Real inv_dt, Real kernel_radius, size_t n, const Point3* positions, const Vector3* velocities, const Real* densities,
                       Vector3* accelerations) = 0;
    sph_force_desc descriptor() const override {
        sph_force_desc d{-1, {}};
        return d;
    }
};
// The same with the complete argument list of NonPressureForce::solve (nonpressure_force.rs:15-27): the context carries the
// materialised fluid-fluid / fluid-boundary contacts (CSR, original index order) and the boundaries (include/sph.h).
struct CustomNonPressureForceWithContacts : NonPressureForce {
    virtual void solve(const sph_host_force_ctx& ctx) = 0;
    sph_force_desc descriptor() const override {
        sph_force_desc d{-2, {}};
        return d;
    }
};
struct XSPHViscosity : NonPressureForce {  // xsph_viscosity.rs:12-26
    Real boundary_viscosity_coefficient, fluid_viscosity_coefficient;
    XSPHViscosity(Real fluid_viscosity_coefficient_, Real boundary_viscosity_coefficient_)
        : boundary_viscosity_coefficient(boundary_viscosity_coefficient_), fluid_viscosity_coefficient(fluid_viscosity_coefficient_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_XSPH_VISCOSITY, {fluid_viscosity_coefficient, boundary_viscosity_coefficient}};
        return d;
    }
};
struct ArtificialViscosity : NonPressureForce {  // artificial_viscosity.rs:14-38
    Real alpha = 1.0f, beta = 0.0f, speed_of_sound = 10.0f, fluid_viscosity_coefficient, boundary_viscosity_coefficient;
    ArtificialViscosity(Real fluid_viscosity_coefficient_, Real boundary_viscosity_coefficient_)
        : fluid_viscosity_coefficient(fluid_viscosity_coefficient_), boundary_viscosity_coefficient(boundary_viscosity_coefficient_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_ARTIFICIAL_VISCOSITY, {fluid_viscosity_coefficient, boundary_viscosity_coefficient, alpha, beta, speed_of_sound}};
        return d;
    }
};
struct Akinci2013SurfaceTension : NonPressureForce {  // akinci2013_surface_tension.rs:20-35
    Real fluid_tension_coefficient, boundary_adhesion_coefficient;
    Akinci2013SurfaceTension(Real fluid_tension_coefficient_, Real boundary_adhesion_coefficient_)
        : fluid_tension_coefficient(fluid_tension_coefficient_), boundary_adhesion_coefficient(boundary_adhesion_coefficient_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_AKINCI2013_TENSION, {fluid_tension_coefficient, boundary_adhesion_coefficient}};
        return d;
    }
};
struct DFSPHViscosity : NonPressureForce {  // dfsph_viscosity.rs:86-124
    size_t min_viscosity_iter = 1, max_viscosity_iter = 50;
    Real max_viscosity_error = 0.01f, viscosity_coefficient;
    explicit DFSPHViscosity(Real viscosity_coefficient_) : viscosity_coefficient(viscosity_coefficient_) {
        if (!(viscosity_coefficient >= 0.0f && viscosity_coefficient <= 1.0f))
            throw std::invalid_argument("The viscosity coefficient must be between 0.0 and 1.0.");  // assert! :106-110
    }
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_DFSPH_VISCOSITY, {viscosity_coefficient, (Real)min_viscosity_iter, (Real)max_viscosity_iter, max_viscosity_error}};
        return d;
    }
};
struct He2014SurfaceTension : NonPressureForce {  // he2014_surface_tension.rs:12-29
    Real fluid_tension_coefficient, boundary_tension_coefficient;
    He2014SurfaceTension(Real fluid_tension_coefficient_, Real boundary_tension_coefficient_)
        : fluid_tension_coefficient(fluid_tension_coefficient_), boundary_tension_coefficient(boundary_tension_coefficient_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_HE2014_TENSION, {fluid_tension_coefficient, boundary_tension_coefficient}};
        return d;
    }
};
struct VorticityConfinement : NonPressureForce {  // no reference counterpart: include/sph.h SPH_FORCE_VORTICITY_CONFINEMENT
    Real eps;  // > 0 and finite, in m/s
    explicit VorticityConfinement(Real eps_) : eps(eps_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_VORTICITY_CONFINEMENT, {eps}};
        return d;
    }
};
struct WCSPHSurfaceTension : NonPressureForce {  // wcsph_surface_tension.rs:15-27 (boundary coefficient must be 0, see sph.h)
    Real fluid_tension_coefficient, boundary_tension_coefficient;
    WCSPHSurfaceTension(Real fluid_tension_coefficient_, Real boundary_tension_coefficient_)
        : fluid_tension_coefficient(fluid_tension_coefficient_), boundary_tension_coefficient(boundary_tension_coefficient_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_WCSPH_TENSION, {fluid_tension_coefficient, boundary_tension_coefficient}};
        return d;
    }
};
struct Becker2009Elasticity : NonPressureForce {  // becker2009_elasticity.rs:60-76
    Real young_modulus, poisson_ratio;
    bool nonlinear_strain;
    Becker2009Elasticity(Real young_modulus_, Real poisson_ratio_, bool nonlinear_strain_)
        : young_modulus(young_modulus_), poisson_ratio(poisson_ratio_), nonlinear_strain(nonlinear_strain_) {}
    sph_force_desc descriptor() const override {
        sph_force_desc d{SPH_FORCE_BECKER2009_ELASTICITY, {young_modulus, poisson_ratio, nonlinear_strain ? 1.0f : 0.0f}};
        return d;
    }
};

// kernel/*.rs: the solver's KernelDensity / KernelGradient type parameters
struct CubicSplineKernel { static constexpr int kind = SPH_KERNEL_CUBIC_SPLINE; };
struct Poly6Kernel { static constexpr int kind = SPH_KERNEL_POLY6; };
struct SpikyKernel { static constexpr int kind = SPH_KERNEL_SPIKY; };
struct ViscosityKernel { static constexpr int kind = SPH_KERNEL_VISCOSITY; };

template <class KernelDensity = CubicSplineKernel, class KernelGradient = CubicSplineKernel>
struct DFSPHSolver {  // dfsph_solver.rs:17-20,54-70
    int kind = SPH_SOLVER_DFSPH;
    int kernel_density = KernelDensity::kind, kernel_gradient = KernelGradient::kind;
    uint32_t min_pressure_iter = 1, max_pressure_iter = 50;
    Real max_density_error = 0.05f;
    uint32_t min_divergence_iter = 1, max_divergence_iter = 50;
    Real max_divergence_error = 0.1f;
    Real omega = 0.5f;
};
template <class KernelDensity = CubicSplineKernel, class KernelGradient = CubicSplineKernel>
struct IISPHSolver : DFSPHSolver<KernelDensity, KernelGradient> {  // iisph_solver.rs:17-20,48-64
    IISPHSolver() { this->kind = SPH_SOLVER_IISPH; }
};

// parry shapes a query can name + the isometry that poses them (liquid_world.rs:246-281)
struct Isometry3 {
    Vector3 translation;
    Real rotation[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};  // row-major
};
struct Ball { Real radius; };
struct Cuboid { Vector3 half_extents; };
struct Capsule { Real half_height, radius; };  // segment along local y
struct Cylinder { Real half_height, radius; };  // axis along local y
struct Cone { Real half_height, radius; };      // axis along local y, apex at (0, half_height, 0), base disc at y = -half_height
// parry HeightField(heights, scale) for ray sampling: nrows x ncols row-major heights, rows along z, columns along x,
// centred on [-0.5, 0.5] * scale in x and z, cells split along their (x0, z1)-(x1, z0) diagonal (DESIGN.md section 11)
struct HeightField {
    uint32_t nrows = 0, ncols = 0;
    std::vector<Real> heights;
    Vector3 scale{1, 1, 1};
};
// the sph_heightfield of a HeightField; it points into s.heights
inline sph_heightfield heightfield_view(const HeightField& s) {
    if (s.heights.size() != (size_t)s.nrows * s.ncols) throw std::runtime_error("salva_b200: HeightField heights must hold nrows * ncols values");
    return sph_heightfield{s.nrows, s.ncols, s.heights.data(), {s.scale.x, s.scale.y, s.scale.z}};
}
// ColliderSampling (fluids_pipeline.rs:64-72): both samplings run on the device
struct ColliderSampling {
    std::vector<Point3> points;  // StaticSampling: in the collider's local frame
    int32_t kind = SPH_SAMPLING_STATIC;
    sph_shape shape{};           // DynamicContactSampling: the collider's shape
    HeightField heightfield;     // ... when shape.kind == SPH_SHAPE_HEIGHTFIELD
    static ColliderSampling StaticSampling(std::vector<Point3> points) { return ColliderSampling{std::move(points)}; }
    static ColliderSampling DynamicContactSampling(const Ball& s) { return contact(sph_shape{SPH_SHAPE_BALL, {s.radius}}); }
    static ColliderSampling DynamicContactSampling(const Cuboid& s) {
        return contact(sph_shape{SPH_SHAPE_CUBOID, {s.half_extents.x, s.half_extents.y, s.half_extents.z}});
    }
    static ColliderSampling DynamicContactSampling(const Capsule& s) { return contact(sph_shape{SPH_SHAPE_CAPSULE, {s.half_height, s.radius}}); }
    static ColliderSampling DynamicContactSampling(const Cylinder& s) { return contact(sph_shape{SPH_SHAPE_CYLINDER, {s.half_height, s.radius}}); }
    static ColliderSampling DynamicContactSampling(const Cone& s) { return contact(sph_shape{SPH_SHAPE_CONE, {s.half_height, s.radius}}); }
    // a heightfield only samples, it never pushes fluid (parry's heightfield point query has is_inside always false)
    static ColliderSampling DynamicContactSampling(const HeightField& s) {
        ColliderSampling c = contact(sph_shape{SPH_SHAPE_HEIGHTFIELD, {}});
        c.heightfield = s;
        return c;
    }

private:
    static ColliderSampling contact(sph_shape shape) {
        ColliderSampling c;
        c.kind = SPH_SAMPLING_CONTACT;
        c.shape = shape;
        return c;
    }
};
using ColliderHandle = uint32_t;

class LiquidWorld;
// trait CouplingManager (coupling/coupling_manager.rs:9-28)
struct CouplingManager {
    virtual ~CouplingManager() {}
    virtual void update_boundaries(LiquidWorld& world, Real dt, Real inv_dt, Real h, Real particle_radius) = 0;
    virtual void transmit_forces(LiquidWorld& world, Real dt, Real inv_dt) = 0;
};

class Fluid {  // object/fluid.rs:12-34
public:
    std::vector<std::shared_ptr<NonPressureForce>> nonpressure_forces;
    std::vector<Point3> positions;
    std::vector<Vector3> velocities;
    std::vector<Real> volumes;
    Real density0;
    InteractionGroups interaction_groups;

    Fluid(std::vector<Point3> particle_positions, Real particle_radius, Real density0_, InteractionGroups groups = InteractionGroups())
        : positions(std::move(particle_positions)), density0(density0_), interaction_groups(groups), particle_radius_(particle_radius) {
        velocities.assign(positions.size(), Vector3());
        volumes.assign(positions.size(), default_particle_volume());
        deleted_.assign(positions.size(), 0);
    }
    size_t num_particles() const { return positions.size(); }
    Real particle_radius() const { return particle_radius_; }
    Real default_particle_volume() const { return particle_radius_ * particle_radius_ * particle_radius_ * (Real)(8.0 * 0.8); }  // fluid.rs:110-120
    Real particle_mass(size_t i) const { return volumes[i] * density0; }                                                           // fluid.rs:183-185
    void add_particles(const std::vector<Point3>& pos, const std::vector<Vector3>* vel = nullptr) {                                // fluid.rs:126-150
        if (vel && vel->size() != pos.size()) throw std::invalid_argument("The provided positions and velocities arrays must have the same length.");
        positions.insert(positions.end(), pos.begin(), pos.end());
        for (size_t i = 0; i < pos.size(); ++i) velocities.push_back(vel ? (*vel)[i] : Vector3());
        volumes.resize(positions.size(), default_particle_volume());
        deleted_.resize(positions.size(), 0);
    }
    void delete_particle_at_next_timestep(size_t particle) {  // fluid.rs:71-76
        if (!deleted_[particle]) {
            deleted_[particle] = 1;
            ++num_deleted_;
        }
    }
    size_t num_deleted_particles() const { return num_deleted_; }

private:
    friend class LiquidWorld;
    Real particle_radius_;
    std::vector<uint8_t> deleted_;
    size_t num_deleted_ = 0;
    size_t n_device_ = 0;                    // particles the engine already holds; positions[n_device_..] are pending appends
    std::vector<Point3> synced_pos_;         // what the engine holds: uploads happen only for real host edits
    std::vector<Vector3> synced_vel_;
    uint32_t handle_ = 0;
    bool alive_ = true;
};

class Boundary {  // object/boundary.rs:11-46
public:
    std::vector<Point3> positions;
    std::vector<Vector3> velocities;
    std::vector<Real> volumes;
    std::vector<Vector3> forces;  // filled after each step when constructed with want_forces (boundary.rs:21)
    InteractionGroups interaction_groups;
    Boundary(std::vector<Point3> particle_positions, InteractionGroups groups = InteractionGroups(), bool want_forces = false)
        : positions(std::move(particle_positions)), interaction_groups(groups), want_forces_(want_forces) {
        velocities.assign(positions.size(), Vector3());
        volumes.assign(positions.size(), 0.0f);
        if (want_forces) forces.assign(positions.size(), Vector3());
    }
    size_t num_particles() const { return positions.size(); }

private:
    friend class LiquidWorld;
    bool want_forces_;
    uint32_t handle_ = 0;
    bool alive_ = true;
    bool coupled_ = false;             // a collider owns the particles: they are read back, never written
    std::vector<Point3> synced_pos_;   // last upload: the engine caches the boundary sort / volumes while they are unchanged
    std::vector<Vector3> synced_vel_;
};

using FluidHandle = size_t;
// A fluid surface mesh (LiquidWorld::extract_surface): counter-clockwise triangles seen from outside, vertex normals when asked
struct SurfaceMesh {
    std::vector<Point3> vertices;
    std::vector<Vector3> normals;
    std::vector<uint32_t> triangles;  // 3 vertex indices per triangle
};
// The anisotropic surface kernels (include/sph.h sph_surface_anisotropy, DESIGN.md section 17); the defaults are
// sph_surface_anisotropy_default's: smoothed centres with round kernels
struct SurfaceAnisotropy {
    Real smoothing = 0.9f;        // lambda in [0, 1]
    Real max_ratio = 1.f;         // k_r in [1, 1000]
    Real isolated_radius = 1.f;   // k_n in [0.001, 1], in units of h
    uint32_t min_neighbours = 6;  // N_eps
};
// One fluid's ellipsoids of the last extraction (LiquidWorld::surface_ellipsoids), in its particle order: per particle the
// centre and 12 floats (e1, a1, e2, a2, e3, a3), a1 >= a2 >= a3
struct SurfaceEllipsoids {
    std::vector<Point3> centres;
    std::vector<Real> axes;
};
// The diffuse particles of a world (LiquidWorld::diffuse), in order; kinds are SPH_DIFFUSE_SPRAY / _FOAM / _BUBBLE
struct DiffuseParticles {
    std::vector<Point3> positions;
    std::vector<Vector3> velocities;
    std::vector<uint8_t> kinds;
    std::vector<Real> lives;
};
using BoundaryHandle = size_t;

class LiquidWorld {  // liquid_world.rs:17-158
public:
    template <class Solver>
    LiquidWorld(const Solver& solver, Real particle_radius, Real smoothing_factor, int device = 0) {
        sph_world_desc d;
        sph_world_desc_default(&d);
        d.solver = solver.kind;
        d.particle_radius = particle_radius;
        d.smoothing_factor = smoothing_factor;
        d.min_pressure_iter = solver.min_pressure_iter;
        d.max_pressure_iter = solver.max_pressure_iter;
        d.max_density_error = solver.max_density_error;
        d.min_divergence_iter = solver.min_divergence_iter;
        d.max_divergence_iter = solver.max_divergence_iter;
        d.max_divergence_error = solver.max_divergence_error;
        d.omega = solver.omega;
        d.kernel_density = solver.kernel_density;
        d.kernel_gradient = solver.kernel_gradient;
        d.device = device;
        sph_status st = sph_world_create(&d, &raw_);
        if (st != SPH_OK) throw std::runtime_error("sph_world_create failed (status " + std::to_string(st) + "): no CUDA device? there is no CPU fallback");
    }
    ~LiquidWorld() {
        if (raw_) sph_world_destroy(raw_);
    }
    LiquidWorld(const LiquidWorld&) = delete;
    LiquidWorld& operator=(const LiquidWorld&) = delete;

    FluidHandle add_fluid(Fluid fluid) {  // liquid_world.rs:161
        uint32_t h = 0;
        check(sph_fluid_add(raw_, fp(fluid.positions), fp(fluid.velocities), fluid.volumes.data(), fluid.positions.size(), fluid.density0,
                            fluid.interaction_groups.memberships, fluid.interaction_groups.filter, &h));
        for (auto& f : fluid.nonpressure_forces) {
            if (auto* custom = dynamic_cast<CustomNonPressureForce*>(f.get())) {  // host callback, kept alive by fluids_
                check(sph_fluid_push_host_force(raw_, h, &LiquidWorld::host_force_trampoline, custom));
                continue;
            }
            if (auto* custom2 = dynamic_cast<CustomNonPressureForceWithContacts*>(f.get())) {
                check(sph_fluid_push_host_force2(raw_, h, &LiquidWorld::host_force_trampoline2, custom2, SPH_HOST_FORCE_CONTACTS | SPH_HOST_FORCE_BOUNDARIES));
                continue;
            }
            sph_force_desc d = f->descriptor();
            check(sph_fluid_push_force(raw_, h, &d));
        }
        fluid.handle_ = h;
        fluid.n_device_ = fluid.positions.size();
        fluid.synced_pos_ = fluid.positions;
        fluid.synced_vel_ = fluid.velocities;
        fluids_.push_back(std::move(fluid));
        return fluids_.size() - 1;
    }
    // liquid_world.rs:171-178: the handle dies, the others stay valid
    void remove_fluid(FluidHandle handle) {
        Fluid& f = fluids_.at(handle);
        if (!f.alive_) throw std::invalid_argument("fluid already removed");
        check(sph_fluid_remove(raw_, f.handle_));
        f.alive_ = false;
        f.positions.clear(); f.velocities.clear(); f.volumes.clear(); f.deleted_.clear();
    }
    void remove_boundary(BoundaryHandle handle) {
        Boundary& b = boundaries_.at(handle);
        if (!b.alive_) throw std::invalid_argument("boundary already removed");
        check(sph_boundary_remove(raw_, b.handle_));
        b.alive_ = false;
        b.positions.clear(); b.velocities.clear(); b.volumes.clear(); b.forces.clear();
    }
    BoundaryHandle add_boundary(Boundary boundary) {  // liquid_world.rs:166
        uint32_t h = 0;
        check(sph_boundary_add(raw_, fp(boundary.positions), fp(boundary.velocities), boundary.positions.size(), boundary.interaction_groups.memberships,
                               boundary.interaction_groups.filter, boundary.want_forces_ ? 1 : 0, &h));
        boundary.handle_ = h;
        boundary.synced_pos_ = boundary.positions;
        boundary.synced_vel_ = boundary.velocities;
        boundaries_.push_back(std::move(boundary));
        return boundaries_.size() - 1;
    }
    std::vector<Fluid>& fluids_mut() { return fluids_; }  // liquid_world.rs:186-188: host edits are uploaded by the next step
    const std::vector<Fluid>& fluids() const { return fluids_; }
    std::vector<Boundary>& boundaries_mut() { return boundaries_; }
    const std::vector<Boundary>& boundaries() const { return boundaries_; }
    Real h() const { return sph_world_h(raw_); }
    Real particle_radius() const { return sph_world_particle_radius(raw_); }
    // CFL-bounded substeps inside each step (sph_world_set_substepping); the defaults are the reference TimestepManager's
    // (timestep_manager.rs:21-31), which has no setter: an extension.  cfl_coeff = 0 turns substepping off.
    void set_substepping(Real cfl_coeff = 0.4f, uint32_t min_substeps = 1, uint32_t max_substeps = 10) {
        check(sph_world_set_substepping(raw_, cfl_coeff, min_substeps, max_substeps));
    }
    // The lengths of the last step's substeps, in order (empty when the step ran no solver).
    std::vector<Real> substeps() {
        size_t n = 0;
        check(sph_world_read_substeps(raw_, nullptr, 0, &n));
        std::vector<Real> out(n);
        if (n) check(sph_world_read_substeps(raw_, out.data(), out.size(), &n));
        return out;
    }

    // Advances the simulation by dt seconds (liquid_world.rs:62-64).
    void step(Real dt, const Vector3& gravity) { step_with_coupling(dt, gravity, nullptr); }
    // n steps of step(dt, gravity) in one call, steps 2..n as one CUDA graph (sph_world_step_many); returns the steps done.
    // On an error it throws as step() does, before the host mirror is pulled.
    uint32_t step_many(Real dt, const Vector3& gravity, uint32_t n) {
        push_host_edits();
        const float g[3] = {gravity.x, gravity.y, gravity.z};
        uint32_t done = 0;
        check(sph_world_step_many(raw_, dt, g, n, &done));
        pull_results();
        return done;
    }
    // Particle sinks and sources applied on the device at the start of every step (sph_fluid_add_sink / sph_fluid_add_source,
    // DESIGN.md section 14): what faucet3.rs:69-105 does with delete_particle_at_next_timestep and add_particles before each
    // step, without reading the fluid.  A sink removes the fluid's particles in [lo, hi) (outside: those not in it); a source
    // appends its template on the first step and every interval-th step after it.  Both return a handle.
    uint32_t add_particle_sink(FluidHandle fluid, const Vector3& lo, const Vector3& hi, bool outside = false) {
        const sph_sink_desc d{{lo.x, lo.y, lo.z}, {hi.x, hi.y, hi.z}, outside ? 1 : 0};
        uint32_t h = 0;
        check(sph_fluid_add_sink(raw_, fluids_.at(fluid).handle_, &d, &h));
        return h;
    }
    uint32_t add_particle_source(FluidHandle fluid, const std::vector<Point3>& pos, const std::vector<Vector3>* vel = nullptr, uint32_t interval = 1) {
        if (vel && vel->size() != pos.size()) throw std::invalid_argument("source positions / velocities differ in length");
        uint32_t h = 0;
        check(sph_fluid_add_source(raw_, fluids_.at(fluid).handle_, fp(pos), vel ? fp(*vel) : nullptr, pos.size(), interval, &h));
        return h;
    }
    void remove_particle_sink(uint32_t sink) { check(sph_sink_remove(raw_, sink)); }
    void remove_particle_source(uint32_t source) { check(sph_source_remove(raw_, source)); }
    // (removed, emitted): the fluid's particles that the last step's sinks removed and its sources emitted
    std::pair<uint32_t, uint32_t> step_edits(FluidHandle fluid) {
        uint32_t r = 0, e = 0;
        check(sph_fluid_read_step_edits(raw_, fluids_.at(fluid).handle_, &r, &e));
        return {r, e};
    }
    // The surface phi = iso of the fluids' smoothed volume fraction (include/sph.h sph_world_extract_surface, DESIGN.md section
    // 15), sampled on a lattice of `spacing` (<= 0: the particle radius).  fluids empty: every fluid.  lo.x > hi.x (the default)
    // meshes the fluids' AABB grown by h, where every surface closes; a box clips the lattice and leaves surfaces open there.
    SurfaceMesh extract_surface(Real iso = 0.6f, Real spacing = 0.f, const std::vector<FluidHandle>& fluids = {}, bool normals = true,
                                const Vector3& lo = Vector3{1, 1, 1}, const Vector3& hi = Vector3{0, 0, 0}) {
        return extract_surface_with(nullptr, iso, spacing, fluids, normals, lo, hi);
    }
    // The same surface with the anisotropic field (include/sph.h sph_world_extract_surface_anisotropic, DESIGN.md section 17):
    // smoothed centres and per-particle ellipsoidal kernels, whose rows surface_ellipsoids reads.
    SurfaceMesh extract_surface(const SurfaceAnisotropy& aniso, Real iso = 0.6f, Real spacing = 0.f, const std::vector<FluidHandle>& fluids = {},
                                bool normals = true, const Vector3& lo = Vector3{1, 1, 1}, const Vector3& hi = Vector3{0, 0, 0}) {
        return extract_surface_with(&aniso, iso, spacing, fluids, normals, lo, hi);
    }
    // The last extraction's ellipsoids of `fluid` (empty after an isotropic extraction or when the fluid was not selected).
    SurfaceEllipsoids surface_ellipsoids(FluidHandle fluid) {
        const uint32_t h = fluids_.at(fluid).handle_;
        size_t n = 0;
        check(sph_world_read_surface_ellipsoids(raw_, h, nullptr, nullptr, 0, &n));
        SurfaceEllipsoids e;
        e.centres.resize(n);
        e.axes.resize(12 * n);
        check(sph_world_read_surface_ellipsoids(raw_, h, reinterpret_cast<float*>(e.centres.data()), e.axes.data(), n, &n));
        return e;
    }
    SurfaceMesh extract_surface_with(const SurfaceAnisotropy* aniso, Real iso, Real spacing, const std::vector<FluidHandle>& fluids, bool normals,
                                     const Vector3& lo, const Vector3& hi) {
        std::vector<uint32_t> hs;
        for (FluidHandle f : fluids) hs.push_back(fluids_.at(f).handle_);
        const sph_surface_desc d{iso, spacing > 0.f ? spacing : particle_radius(), {lo.x, lo.y, lo.z}, {hi.x, hi.y, hi.z}, normals ? 1 : 0};
        size_t nv = 0, nt = 0;
        if (aniso) {
            const sph_surface_anisotropy a{aniso->smoothing, aniso->max_ratio, aniso->isolated_radius, aniso->min_neighbours};
            check(sph_world_extract_surface_anisotropic(raw_, hs.data(), hs.size(), &d, &a, &nv, &nt));
        } else {
            check(sph_world_extract_surface(raw_, hs.data(), hs.size(), &d, &nv, &nt));
        }
        SurfaceMesh m;
        m.vertices.resize(nv);
        m.normals.resize(normals ? nv : 0);
        m.triangles.resize(3 * nt);
        check(sph_world_read_surface(raw_, reinterpret_cast<float*>(m.vertices.data()), normals ? reinterpret_cast<float*>(m.normals.data()) : nullptr, nv,
                                     m.triangles.data(), nt));
        return m;
    }
    // Advances the diffuse set (spray, foam, air bubbles: include/sph.h sph_world_update_diffuse, DESIGN.md section 16) by one
    // frame of length dt from `fluids` (empty: every fluid).  desc: sph_diffuse_desc_default's values when not given.
    sph_diffuse_stats update_diffuse(Real dt, const Vector3& gravity, const sph_diffuse_desc* desc = nullptr,
                                     const std::vector<FluidHandle>& fluids = {}) {
        std::vector<uint32_t> hs;
        for (FluidHandle f : fluids) hs.push_back(fluids_.at(f).handle_);
        sph_diffuse_desc d;
        sph_diffuse_desc_default(&d);
        if (desc) d = *desc;
        const float g[3] = {gravity.x, gravity.y, gravity.z};
        sph_diffuse_stats st;
        check(sph_world_update_diffuse(raw_, hs.data(), hs.size(), &d, dt, g, &st));
        return st;
    }
    DiffuseParticles diffuse() {
        size_t n = 0;
        check(sph_world_read_diffuse(raw_, nullptr, nullptr, nullptr, nullptr, 0, &n));
        DiffuseParticles p;
        p.positions.resize(n);
        p.velocities.resize(n);
        p.kinds.resize(n);
        p.lives.resize(n);
        check(sph_world_read_diffuse(raw_, reinterpret_cast<float*>(p.positions.data()), reinterpret_cast<float*>(p.velocities.data()),
                                     p.kinds.data(), p.lives.data(), n, &n));
        return p;
    }
    // liquid_world.rs:67-158
    void step_with_coupling(Real dt, const Vector3& gravity, CouplingManager* coupling) {
        push_host_edits();
        const float g[3] = {gravity.x, gravity.y, gravity.z};
        if (coupling) {
            CouplingCtx ctx{this, coupling};
            sph_coupling_manager cm{&LiquidWorld::coupling_update, &LiquidWorld::coupling_transmit, &ctx};
            check(sph_world_step_with_coupling(raw_, dt, g, &cm));
        } else {
            check(sph_world_step(raw_, dt, g));  // == LiquidWorld::step
        }
        pull_results();
    }
    // Host edits made through fluids_mut() / boundaries_mut() since the last sync go to the engine; unchanged arrays are
    // NOT re-uploaded (the engine reuses its boundary sort and volumes while boundaries are untouched).
    void push_host_edits() {
        for (Fluid& f : fluids_) {
            if (!f.alive_) continue;
            if (f.velocities.size() != f.positions.size()) throw std::invalid_argument("fluid positions / velocities differ in length");
            const size_t n_dev = f.n_device_;
            if (f.positions.size() < n_dev) throw std::invalid_argument("delete particles with delete_particle_at_next_timestep, not by shrinking the arrays");
            if (n_dev && (!same(f.positions, f.synced_pos_, n_dev) || !same(f.velocities, f.synced_vel_, n_dev)))
                check(sph_fluid_write(raw_, f.handle_, fp(f.positions), fp(f.velocities), n_dev));
            if (f.positions.size() > n_dev) {  // Fluid::add_particles: appended from the LIVE tail, so later edits of the tail count
                check(sph_fluid_append(raw_, f.handle_, fp(f.positions) + 3 * n_dev, fp(f.velocities) + 3 * n_dev, f.positions.size() - n_dev));
                f.n_device_ = f.positions.size();
            }
            if (f.num_deleted_) {
                check(sph_fluid_delete(raw_, f.handle_, f.deleted_.data(), f.deleted_.size()));
                f.num_deleted_ = 0;
            }
        }
        for (Boundary& b : boundaries_) {
            if (!b.alive_ || b.coupled_) continue;
            if (b.velocities.size() != b.positions.size()) b.velocities.resize(b.positions.size());
            if (b.positions.size() != b.synced_pos_.size()) {
                check(sph_boundary_set_particles(raw_, b.handle_, fp(b.positions), fp(b.velocities), b.positions.size()));
            } else if (b.num_particles() && (!same(b.positions, b.synced_pos_, b.num_particles()) || !same(b.velocities, b.synced_vel_, b.num_particles()))) {
                check(sph_boundary_write(raw_, b.handle_, fp(b.positions), fp(b.velocities), b.num_particles()));
            } else {
                continue;
            }
            b.synced_pos_ = b.positions;
            b.synced_vel_ = b.velocities;
            b.volumes.resize(b.positions.size(), 0.0f);
            if (b.want_forces_) b.forces.resize(b.positions.size());
        }
    }
    void pull_results() {
        for (Fluid& f : fluids_) {
            if (!f.alive_) continue;
            size_t n = 0;
            check(sph_fluid_count(raw_, f.handle_, &n));
            f.positions.resize(n);
            f.velocities.resize(n);
            f.volumes.resize(n, f.default_particle_volume());
            f.deleted_.assign(n, 0);
            if (n) check(sph_fluid_read(raw_, f.handle_, reinterpret_cast<float*>(f.positions.data()), reinterpret_cast<float*>(f.velocities.data()), n, &n));
            f.n_device_ = n;
            f.synced_pos_ = f.positions;
            f.synced_vel_ = f.velocities;
        }
        for (Boundary& b : boundaries_) {
            if (!b.alive_) continue;
            if (b.coupled_) {  // boundary.positions / velocities as the collider posed them
                size_t n = 0;
                check(sph_boundary_read(raw_, b.handle_, nullptr, nullptr, 0, &n));
                b.positions.resize(n);
                b.velocities.resize(n);
                b.volumes.resize(n);
                b.forces.resize(n);
                if (n) check(sph_boundary_read(raw_, b.handle_, reinterpret_cast<float*>(b.positions.data()), reinterpret_cast<float*>(b.velocities.data()), n, &n));
                b.synced_pos_ = b.positions;
                b.synced_vel_ = b.velocities;
            }
            if (!b.num_particles()) continue;
            check(sph_boundary_read_volumes(raw_, b.handle_, b.volumes.data(), b.volumes.size()));
            if (b.coupled_) check(sph_boundary_read_forces(raw_, b.handle_, reinterpret_cast<float*>(b.forces.data()), b.forces.size()));
            else if (b.want_forces_) check(sph_boundary_read_forces(raw_, b.handle_, reinterpret_cast<float*>(b.forces.data()), b.forces.size()));
        }
    }
    // Snapshot / restore of the state the solver carries across steps (include/sph.h sph_world_snapshot_*).
    std::vector<char> snapshot() {
        push_host_edits();
        size_t n = 0, wr = 0;
        check(sph_world_snapshot_size(raw_, &n));
        std::vector<char> blob(n);
        check(sph_world_snapshot_save(raw_, blob.data(), blob.size(), &wr));
        blob.resize(wr);
        return blob;
    }
    void restore(const std::vector<char>& blob) {
        check(sph_world_snapshot_load(raw_, blob.data(), blob.size()));
        pull_results();
    }
    // liquid_world.rs:211-243 (ParticleId::FluidParticle(handle, i) / BoundaryParticle(handle, i)), sorted.
    struct ParticleId {
        bool is_boundary;
        uint32_t handle, index;
    };
    std::vector<ParticleId> particles_intersecting_aabb(const Point3& mins, const Point3& maxs) {
        const float lo[3] = {mins.x, mins.y, mins.z}, hi[3] = {maxs.x, maxs.y, maxs.z};
        std::vector<uint32_t> k(256), h(256), i(256);
        size_t n = 0;
        for (;;) {
            check(sph_world_particles_in_aabb(raw_, lo, hi, k.data(), h.data(), i.data(), k.size(), &n));
            if (n <= k.size()) break;
            k.resize(n); h.resize(n); i.resize(n);
        }
        std::vector<ParticleId> out(n);
        for (size_t t = 0; t < n; ++t) out[t] = ParticleId{k[t] != 0, h[t], i[t]};
        return out;
    }
    // liquid_world.rs:246-281 for Ball / Cuboid / Capsule / Cylinder / Cone / HeightField
    // ray_sampling.rs:9-24 on this world's device (salva3d::sampling below): points in ascending quantised-key order
    std::vector<Point3> ray_sample(int32_t method, const sph_shape& shape, const sph_heightfield* hf, Real particle_rad) {
        std::vector<Point3> out(4096);
        size_t n = 0;
        for (;;) {
            check(sph_world_sample_shape(raw_, method, &shape, hf, particle_rad, reinterpret_cast<float*>(out.data()), out.size(), &n));
            if (n <= out.size()) break;
            out.resize(n);
        }
        out.resize(n);
        return out;
    }
    std::vector<ParticleId> particles_intersecting_shape(const Isometry3& pos, const Ball& s) { return shape_query(pos, sph_shape{SPH_SHAPE_BALL, {s.radius}}); }
    std::vector<ParticleId> particles_intersecting_shape(const Isometry3& pos, const Cuboid& s) {
        return shape_query(pos, sph_shape{SPH_SHAPE_CUBOID, {s.half_extents.x, s.half_extents.y, s.half_extents.z}});
    }
    std::vector<ParticleId> particles_intersecting_shape(const Isometry3& pos, const Capsule& s) {
        return shape_query(pos, sph_shape{SPH_SHAPE_CAPSULE, {s.half_height, s.radius}});
    }
    std::vector<ParticleId> particles_intersecting_shape(const Isometry3& pos, const Cylinder& s) {
        return shape_query(pos, sph_shape{SPH_SHAPE_CYLINDER, {s.half_height, s.radius}});
    }
    std::vector<ParticleId> particles_intersecting_shape(const Isometry3& pos, const Cone& s) {
        return shape_query(pos, sph_shape{SPH_SHAPE_CONE, {s.half_height, s.radius}});
    }
    std::vector<ParticleId> particles_intersecting_shape(const Isometry3& pos, const HeightField& s) {
        const sph_heightfield hf = heightfield_view(s);
        return shape_query(pos, [&](const float* t, uint32_t* k, uint32_t* h, uint32_t* i, size_t cap, size_t* n) {
            return sph_world_particles_in_heightfield(raw_, &hf, t, pos.rotation, k, h, i, cap, n);
        });
    }
    // ColliderCouplingSet::register_coupling fluids_pipeline.rs:98-114: the boundary's particles become the collider's samples
    // (DynamicContactSampling: from the next step on, its size changes every step)
    ColliderHandle register_coupling(BoundaryHandle boundary, const ColliderSampling& sampling) {
        Boundary& b = boundaries_.at(boundary);
        uint32_t c = 0;
        if (sampling.kind == SPH_SAMPLING_CONTACT && sampling.shape.kind == SPH_SHAPE_HEIGHTFIELD) {
            const sph_heightfield hf = heightfield_view(sampling.heightfield);
            check(sph_collider_register_heightfield(raw_, b.handle_, &hf, &c));
        } else {
            check(sph_collider_register(raw_, b.handle_, sampling.kind, sampling.kind == SPH_SAMPLING_CONTACT ? &sampling.shape : nullptr,
                                        fp(sampling.points), sampling.points.size(), &c));
        }
        b.coupled_ = true;
        pull_results();
        return c;
    }
    // collider.position() and its parent body for the next steps (SPH_BODY_NONE / _FIXED / _DYNAMIC)
    void set_collider_state(ColliderHandle c, const Isometry3& pos, int body, const Vector3& linvel = Vector3(), const Vector3& angvel = Vector3(),
                            const Point3& world_com = Point3()) {
        sph_collider_state s;
        s.translation[0] = pos.translation.x; s.translation[1] = pos.translation.y; s.translation[2] = pos.translation.z;
        std::memcpy(s.rotation_rowmajor, pos.rotation, sizeof s.rotation_rowmajor);
        s.body = body;
        s.linvel[0] = linvel.x; s.linvel[1] = linvel.y; s.linvel[2] = linvel.z;
        s.angvel[0] = angvel.x; s.angvel[1] = angvel.y; s.angvel[2] = angvel.z;
        s.world_com[0] = world_com.x; s.world_com[1] = world_com.y; s.world_com[2] = world_com.z;
        check(sph_collider_set_state(raw_, c, &s));
    }
    // transmit_forces fluids_pipeline.rs:263-287: (linear, angular) impulse of the last step
    std::pair<Vector3, Vector3> collider_impulse(ColliderHandle c) {
        float lin[3], ang[3];
        check(sph_collider_read_impulse(raw_, c, lin, ang));
        return {Vector3{lin[0], lin[1], lin[2]}, Vector3{ang[0], ang[1], ang[2]}};
    }
    // ColliderCouplingSet::unregister_coupling fluids_pipeline.rs:119-122: the boundary stays with its last particles
    void unregister_coupling(ColliderHandle c, BoundaryHandle boundary) {
        check(sph_collider_unregister(raw_, c));
        boundaries_.at(boundary).coupled_ = false;
    }
    sph_step_stats counters() const {  // world.counters (counters/mod.rs:17-30)
        sph_step_stats s;
        sph_world_stats(raw_, &s);
        return s;
    }
    sph_world* raw() { return raw_; }

private:
    static void host_force_trampoline(void* user, float dt, float inv_dt, float kernel_radius, size_t n, const float* pos, const float* vel,
                                      const float* dens, float* acc) {
        static_cast<CustomNonPressureForce*>(user)->solve(dt, inv_dt, kernel_radius, n, reinterpret_cast<const Point3*>(pos),
                                                          reinterpret_cast<const Vector3*>(vel), dens, reinterpret_cast<Vector3*>(acc));
    }
    static void host_force_trampoline2(void* user, const sph_host_force_ctx* ctx) { static_cast<CustomNonPressureForceWithContacts*>(user)->solve(*ctx); }
    struct CouplingCtx {
        LiquidWorld* world;
        CouplingManager* manager;
    };
    // update_boundaries sees the mirror's host arrays: pull the fluids first, push the callback's edits back afterwards
    static void coupling_update(void* user, sph_world*, float dt, float inv_dt, float h, float particle_radius) {
        auto* c = static_cast<CouplingCtx*>(user);
        c->world->pull_results();
        c->manager->update_boundaries(*c->world, dt, inv_dt, h, particle_radius);
        c->world->push_host_edits();
    }
    static void coupling_transmit(void* user, sph_world*, float dt, float inv_dt) {
        auto* c = static_cast<CouplingCtx*>(user);
        c->world->pull_results();
        c->manager->transmit_forces(*c->world, dt, inv_dt);
    }
    std::vector<ParticleId> shape_query(const Isometry3& pos, sph_shape shape) {
        return shape_query(pos, [&](const float* t, uint32_t* k, uint32_t* h, uint32_t* i, size_t cap, size_t* n) {
            return sph_world_particles_in_shape(raw_, &shape, t, pos.rotation, k, h, i, cap, n);
        });
    }
    template <class Query>
    std::vector<ParticleId> shape_query(const Isometry3& pos, Query query) {
        const float t[3] = {pos.translation.x, pos.translation.y, pos.translation.z};
        std::vector<uint32_t> k(256), h(256), i(256);
        size_t n = 0;
        for (;;) {
            check(query(t, k.data(), h.data(), i.data(), k.size(), &n));
            if (n <= k.size()) break;
            k.resize(n); h.resize(n); i.resize(n);
        }
        std::vector<ParticleId> out(n);
        for (size_t q = 0; q < n; ++q) out[q] = ParticleId{k[q] != 0, h[q], i[q]};
        return out;
    }
    template <class V>
    static bool same(const std::vector<V>& a, const std::vector<V>& b, size_t n) {
        return a.size() >= n && b.size() >= n && (n == 0 || std::memcmp(a.data(), b.data(), n * sizeof(V)) == 0);
    }
    template <class V>
    static const float* fp(const std::vector<V>& v) {
        static_assert(sizeof(V) == 3 * sizeof(float), "packed xyz triples");
        return v.empty() ? nullptr : reinterpret_cast<const float*>(v.data());
    }
    void check(sph_status st) const {  // reference assert!/panic sites surface as exceptions
        if (st != SPH_OK) throw std::runtime_error(std::string("salva_b200: status ") + std::to_string((int)st) + ": " + sph_last_error(raw_));
    }
    sph_world* raw_ = nullptr;
    std::vector<Fluid> fluids_;
    std::vector<Boundary> boundaries_;
};

// salva3d::sampling (sampling/ray_sampling.rs:9-24).  The world is the one extra argument: its device runs the sampler.
namespace sampling {
namespace detail {
inline std::vector<Point3> run(LiquidWorld& w, int32_t m, const Ball& s, Real r) { return w.ray_sample(m, sph_shape{SPH_SHAPE_BALL, {s.radius}}, nullptr, r); }
inline std::vector<Point3> run(LiquidWorld& w, int32_t m, const Cuboid& s, Real r) {
    return w.ray_sample(m, sph_shape{SPH_SHAPE_CUBOID, {s.half_extents.x, s.half_extents.y, s.half_extents.z}}, nullptr, r);
}
inline std::vector<Point3> run(LiquidWorld& w, int32_t m, const Capsule& s, Real r) {
    return w.ray_sample(m, sph_shape{SPH_SHAPE_CAPSULE, {s.half_height, s.radius}}, nullptr, r);
}
inline std::vector<Point3> run(LiquidWorld& w, int32_t m, const Cylinder& s, Real r) {
    return w.ray_sample(m, sph_shape{SPH_SHAPE_CYLINDER, {s.half_height, s.radius}}, nullptr, r);
}
inline std::vector<Point3> run(LiquidWorld& w, int32_t m, const Cone& s, Real r) {
    return w.ray_sample(m, sph_shape{SPH_SHAPE_CONE, {s.half_height, s.radius}}, nullptr, r);
}
inline std::vector<Point3> run(LiquidWorld& w, int32_t m, const HeightField& s, Real r) {
    const sph_heightfield hf = heightfield_view(s);
    return w.ray_sample(m, sph_shape{SPH_SHAPE_HEIGHTFIELD, {}}, &hf, r);
}
}  // namespace detail
template <class S>
std::vector<Point3> shape_surface_ray_sample(LiquidWorld& world, const S& shape, Real particle_rad) {
    return detail::run(world, SPH_SAMPLE_SURFACE, shape, particle_rad);
}
template <class S>
std::vector<Point3> shape_volume_ray_sample(LiquidWorld& world, const S& shape, Real particle_rad) {
    return detail::run(world, SPH_SAMPLE_VOLUME, shape, particle_rad);
}
}  // namespace sampling

}  // namespace salva3d
