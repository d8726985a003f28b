"""Host-side mirror of salva3d's solver-path API on top of the C ABI (include/sph.h).

The reference toolchain (Rust) is absent here, so the host side above the C ABI is this thin Python
mirror with the reference's names and argument meaning (the Rust shim a maintainer would add is in
INTEGRATION.md).  Mirrors:
  LiquidWorld::{new, step, add_fluid, add_boundary, h, particle_radius}   liquid_world.rs:39-208
  Fluid::{new, add_particles, delete_particle_at_next_timestep, num_particles}  fluid.rs:40-185
  Boundary::new                                                           boundary.rs:28-46
  DFSPHSolver::new / IISPHSolver::new (public tunables)                   dfsph_solver.rs:54-70, iisph_solver.rs:48-64
  XSPHViscosity / ArtificialViscosity / Akinci2013SurfaceTension / Becker2009Elasticity ::new
Every call goes to the CUDA library; there is no CPU path.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import ForceDesc, StepStats, WorldDesc

DBG = dict(density=0, alpha=1, divergence=2, predicted_density=3, velocity_change=4, num_fluid_contacts=5,
           num_boundary_contacts=6, pressure=7, acceleration=8, dii=9, aii=10, dij_pjl=11, he2014_color=12, he2014_gradc=13,
           visc_beta=14, visc_target=15, el_volume0=16, el_rotation=17, el_grad_tr=18, el_stress=19, diffuse_normal=20,
           diffuse_trapped_air=21, diffuse_wave_crest=22, diffuse_kinetic=23, diffuse_count=24,
           fluid_list_bits=25, vorticity=26, vorticity_eta=27)
# floats per particle of the selectors that are not scalars (include/sph.h)
WIDTH = {4: 3, 8: 3, 9: 3, 11: 3, 14: 36, 15: 6, 17: 9, 18: 9, 19: 6, 20: 3, 26: 3, 27: 3}
DIFFUSE_KINDS = ("spray", "foam", "bubble")  # SPH_DIFFUSE_SPRAY / _FOAM / _BUBBLE


class SphError(RuntimeError):
    """A non-OK sph_status; reference assertion sites surface here (the Rust shim re-panics)."""

    def __init__(self, status, message):
        super().__init__("%s: %s" % (_lib.STATUS_NAMES.get(status, status), message))
        self.status = status


class SurfaceAnisotropy:
    """include/sph.h sph_surface_anisotropy (Yu & Turk 2013 kernels, DESIGN.md section 17): centre smoothing lambda in [0, 1],
    largest semi-axis ratio k_r in [1, 1000], radius of a particle with too few neighbours k_n in [0.001, 1] (units of h),
    and the fewest neighbours N_eps for an anisotropic kernel.  The defaults are sph_surface_anisotropy_default's: smoothed
    centres with round kernels (k_r = k_n = 1); k_r > 1 stretches the kernels, see DESIGN.md section 17 for its cost."""

    def __init__(self, smoothing=0.9, max_ratio=1.0, isolated_radius=1.0, min_neighbours=6):
        self.smoothing, self.max_ratio = smoothing, max_ratio
        self.isolated_radius, self.min_neighbours = isolated_radius, min_neighbours

    def _c(self):
        return _lib.SurfaceAnisotropy(float(self.smoothing), float(self.max_ratio), float(self.isolated_radius), int(self.min_neighbours))


class InteractionGroups:
    """interaction_groups.rs:20-79; default = (GROUP_1, ALL)."""

    def __init__(self, memberships=1, filter=0xFFFFFFFF):
        self.memberships, self.filter = memberships, filter

    def test(self, rhs):
        return (self.memberships & rhs.filter) != 0 and (rhs.memberships & self.filter) != 0


class CubicSplineKernel:
    """kernel/cubic_spline_kernel.rs"""
    kind = 0


class Poly6Kernel:
    """kernel/poly6_kernel.rs"""
    kind = 1


class SpikyKernel:
    """kernel/spiky_kernel.rs"""
    kind = 2


class ViscosityKernel:
    """kernel/viscosity_kernel.rs"""
    kind = 3


class DFSPHSolver:
    """dfsph_solver.rs:54-70 defaults; DFSPHSolver<KernelDensity, KernelGradient> (dfsph_solver.rs:17-20) as constructor arguments."""
    kind = 0

    def __init__(self, kernel_density=CubicSplineKernel, kernel_gradient=CubicSplineKernel):
        self.kernel_density, self.kernel_gradient = kernel_density.kind, kernel_gradient.kind
        self.min_pressure_iter, self.max_pressure_iter, self.max_density_error = 1, 50, 0.05
        self.min_divergence_iter, self.max_divergence_iter, self.max_divergence_error = 1, 50, 0.1
        self.omega = 0.5


class IISPHSolver(DFSPHSolver):
    """iisph_solver.rs:48-64 defaults."""
    kind = 1


class XSPHViscosity:
    kind = 0

    def __init__(self, fluid_viscosity_coefficient, boundary_viscosity_coefficient):
        self.params = [fluid_viscosity_coefficient, boundary_viscosity_coefficient]


class ArtificialViscosity:
    kind = 1

    def __init__(self, fluid_viscosity_coefficient, boundary_viscosity_coefficient, alpha=1.0, beta=0.0,
                 speed_of_sound=10.0):
        self.params = [fluid_viscosity_coefficient, boundary_viscosity_coefficient, alpha, beta, speed_of_sound]


class Akinci2013SurfaceTension:
    kind = 2

    def __init__(self, fluid_tension_coefficient, boundary_adhesion_coefficient):
        self.params = [fluid_tension_coefficient, boundary_adhesion_coefficient]


class Becker2009Elasticity:
    kind = 3

    def __init__(self, young_modulus, poisson_ratio, nonlinear_strain):
        self.params = [young_modulus, poisson_ratio, 1.0 if nonlinear_strain else 0.0]


class DFSPHViscosity:
    """dfsph_viscosity.rs:86-124 (public tunables min/max_viscosity_iter, max_viscosity_error)"""
    kind = 6

    def __init__(self, viscosity_coefficient, min_viscosity_iter=1, max_viscosity_iter=50, max_viscosity_error=0.01):
        if not 0.0 <= viscosity_coefficient <= 1.0:
            raise ValueError("The viscosity coefficient must be between 0.0 and 1.0.")
        self.viscosity_coefficient = viscosity_coefficient
        self.min_viscosity_iter = min_viscosity_iter
        self.max_viscosity_iter = max_viscosity_iter
        self.max_viscosity_error = max_viscosity_error

    @property
    def params(self):
        return [self.viscosity_coefficient, float(self.min_viscosity_iter), float(self.max_viscosity_iter), self.max_viscosity_error]


class He2014SurfaceTension:
    """he2014_surface_tension.rs:21-29"""
    kind = 4

    def __init__(self, fluid_tension_coefficient, boundary_tension_coefficient):
        self.params = [fluid_tension_coefficient, boundary_tension_coefficient]


class VorticityConfinement:
    """Vorticity confinement, a_i += eps (N_i x omega_i) with eps > 0 in m/s (include/sph.h SPH_FORCE_VORTICITY_CONFINEMENT,
    DESIGN.md section 18); no reference counterpart"""
    kind = 7

    def __init__(self, eps):
        self.params = [eps]


class WCSPHSurfaceTension:
    """wcsph_surface_tension.rs:21-27; a non-zero boundary coefficient is rejected (include/sph.h SPH_FORCE_WCSPH_TENSION)"""
    kind = 5

    def __init__(self, fluid_tension_coefficient, boundary_tension_coefficient):
        self.params = [fluid_tension_coefficient, boundary_tension_coefficient]


class Ball:
    """parry Ball(radius) for particles_intersecting_shape"""
    kind = 1

    def __init__(self, radius):
        self.params = [radius]


class Cuboid:
    """parry Cuboid(half_extents)"""
    kind = 2

    def __init__(self, half_extents):
        self.params = list(half_extents)


class Capsule:
    """parry Capsule along local y: half_height, radius"""
    kind = 3

    def __init__(self, half_height, radius):
        self.params = [half_height, radius]


class Cylinder:
    """parry Cylinder along local y: half_height, radius (sqrt(x^2 + z^2) <= radius, |y| <= half_height)"""
    kind = 5

    def __init__(self, half_height, radius):
        self.params = [half_height, radius]


class Cone:
    """parry Cone along local y: half_height, base radius; the apex at (0, half_height, 0), the base disc at y = -half_height"""
    kind = 6

    def __init__(self, half_height, radius):
        self.params = [half_height, radius]


class StaticSampling:
    """ColliderSampling::StaticSampling(points) (fluids_pipeline.rs:64-69): the collider approximated by sample points given
    in its local frame."""
    kind = 0

    def __init__(self, points):
        self.points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)


class DynamicContactSampling:
    """ColliderSampling::DynamicContactSampling (fluids_pipeline.rs:71, 192-255): every step the collider's shape (Ball,
    Cuboid, Capsule, Cylinder, Cone or sampling.HeightField) is sampled where the fluid is about to touch it, and penetrating fluid particles
    are pushed out.  A heightfield never pushes (parry's heightfield point query has is_inside always false): it only samples."""
    kind = 1

    def __init__(self, shape):
        self.shape = shape


HEIGHTFIELD = 4  # SPH_SHAPE_HEIGHTFIELD: salva_b200.sampling.HeightField


def heightfield_c(shape):
    """The sph_heightfield of a sampling.HeightField; it points into shape.heights, which must outlive the call."""
    hf = _lib.HeightFieldC()
    hf.nrows, hf.ncols = shape.heights.shape
    hf.heights = shape.heights.ctypes.data_as(C.POINTER(C.c_float))
    hf.scale[:] = shape.scale
    return hf


# the rigid body a collider is attached to (include/sph.h SPH_BODY_*)
BODY_NONE, BODY_FIXED, BODY_DYNAMIC = 0, 1, 2


class CouplingManager:
    """trait CouplingManager (coupling/coupling_manager.rs:9-28).  Subclass and override; `world` is the LiquidWorld being
    stepped (queries issued from update_boundaries see fluid particles only, liquid_world.rs:86-103)."""

    def update_boundaries(self, world, dt, inv_dt, h, particle_radius):
        pass

    def transmit_forces(self, world, dt, inv_dt):
        pass


class ContactsView:
    """ParticlesContacts (contacts.rs:83-121) of one fluid as CSR numpy views: offsets (n+1), j, j_model, weight, gradient (m, 3)."""

    def __init__(self, offsets, j, j_model, weight, gradient):
        self.offsets, self.j, self.j_model, self.weight, self.gradient = offsets, j, j_model, weight, gradient

    def particle_contacts(self, i):
        """contacts.rs:107-110: slice of particle i's contacts"""
        return slice(int(self.offsets[i]), int(self.offsets[i + 1]))


class Fluid:
    """fluid.rs:12-68: host description handed to LiquidWorld.add_fluid."""

    def __init__(self, particle_positions, particle_radius, density0, interaction_groups=None):
        self.positions = np.ascontiguousarray(particle_positions, np.float32).reshape(-1, 3)
        self.velocities = None
        self.volumes = None
        self.particle_radius = particle_radius
        self.density0 = density0
        self.interaction_groups = interaction_groups or InteractionGroups()
        self.nonpressure_forces = []

    def num_particles(self):
        return len(self.positions)


class Boundary:
    """boundary.rs:11-46"""

    def __init__(self, particle_positions, interaction_groups=None, want_forces=False):
        self.positions = np.ascontiguousarray(particle_positions, np.float32).reshape(-1, 3)
        self.velocities = None
        self.interaction_groups = interaction_groups or InteractionGroups()
        self.want_forces = want_forces


def _f32(a, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a.reshape(shape) if shape is not None else a


def _fp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def _view(ptr, shape, dtype=np.float32):
    """numpy view of a callback's pointer argument; an empty one (an empty fluid's, possibly NULL) as an empty array."""
    n = int(np.prod(shape))
    if n == 0 or not ptr:
        return np.zeros(shape, dtype)
    return np.ctypeslib.as_array(ptr, (n,)).view(dtype).reshape(shape)


def nccl_unique_id():
    """128-byte NCCL unique id (rank 0 creates it, the host's plumbing broadcasts it)."""
    buf = C.create_string_buffer(128)
    st = _lib.lib().sph_nccl_unique_id(buf)
    if st != 0:
        raise SphError(st, "sph_nccl_unique_id failed (libnccl not loadable?)")
    return buf.raw


class LiquidWorld:
    """liquid_world.rs:17-158 on the GPU engine."""

    def __init__(self, solver=None, particle_radius=0.05, smoothing_factor=2.0, device=0, deterministic=True,
                 slab_rank=0, slab_count=1, gather_backend=0):
        solver = solver or DFSPHSolver()
        # the solver's kernels are compile-time parameters (dfsph_solver.rs:17-20): non-default ones live in the second library
        self._L = _lib.lib(kernels=bool(getattr(solver, "kernel_density", 0) or getattr(solver, "kernel_gradient", 0)))
        d = WorldDesc()
        self._L.sph_world_desc_default(C.byref(d))
        d.solver = solver.kind
        d.particle_radius = particle_radius
        d.smoothing_factor = smoothing_factor
        d.min_pressure_iter, d.max_pressure_iter = solver.min_pressure_iter, solver.max_pressure_iter
        d.max_density_error = solver.max_density_error
        d.min_divergence_iter, d.max_divergence_iter = solver.min_divergence_iter, solver.max_divergence_iter
        d.max_divergence_error = solver.max_divergence_error
        d.omega = solver.omega
        d.device = device
        d.deterministic = int(deterministic)
        d.slab_rank, d.slab_count = slab_rank, slab_count
        d.gather_backend = gather_backend  # must be 0 (the only gather backend); sph_world_create refuses other values
        d.kernel_density = getattr(solver, "kernel_density", 0)
        d.kernel_gradient = getattr(solver, "kernel_gradient", 0)
        self._w = C.c_void_p()
        st = self._L.sph_world_create(C.byref(d), C.byref(self._w))
        if st != 0:
            self._w = None
            raise SphError(st, "sph_world_create failed (no CUDA device?); there is no CPU fallback")
        self._nb = {}
        self._callbacks = []

    def close(self):
        if getattr(self, "_w", None):
            self._L.sph_world_destroy(self._w)
            self._w = None

    def __del__(self):
        self.close()

    def _ck(self, st):
        if st != 0:
            raise SphError(st, self._L.sph_last_error(self._w).decode())

    # -- reference-shaped API ------------------------------------------------------------------
    @property
    def h(self):
        return self._L.sph_world_h(self._w)

    @property
    def particle_radius(self):
        return self._L.sph_world_particle_radius(self._w)

    def add_fluid(self, fluid_or_positions, density0=1000.0, velocities=None, volumes=None, memberships=1,
                  filter=0xFFFFFFFF):
        forces = []
        if isinstance(fluid_or_positions, Fluid):
            f = fluid_or_positions
            p, velocities, volumes, density0 = f.positions, f.velocities, f.volumes, f.density0
            memberships, filter = f.interaction_groups.memberships, f.interaction_groups.filter
            forces = f.nonpressure_forces
        else:
            p = fluid_or_positions
        p = _f32(p, (-1, 3))
        v = _f32(velocities, (-1, 3))
        vol = _f32(volumes)
        h = C.c_uint32()
        self._ck(self._L.sph_fluid_add(self._w, _fp(p), _fp(v), _fp(vol), len(p), density0, memberships, filter,
                                       C.byref(h)))
        for fo in forces:
            self.push_force(h.value, fo.kind, fo.params)
        return h.value

    def push_force(self, fluid, kind, params):
        d = ForceDesc()
        d.kind = kind
        for i, x in enumerate(params):
            d.p[i] = x
        self._ck(self._L.sph_fluid_push_force(self._w, fluid, C.byref(d)))

    def push_host_force(self, fluid, solve):
        """User-defined NonPressureForce (nonpressure_force.rs:10-30): solve(dt, inv_dt, kernel_radius, positions,
        velocities, densities, accelerations) is called on the host with numpy views in ORIGINAL index order and adds
        to `accelerations` in place (examples3d/custom_forces3.rs:66-90)."""
        def tramp(_user, dt, inv_dt, h, n, pos, vel, dens, acc):
            solve(dt, inv_dt, h, _view(pos, (n, 3)), _view(vel, (n, 3)), _view(dens, (n,)), _view(acc, (n, 3)))
        cb = _lib.HOST_FORCE_FN(tramp)
        self._callbacks.append(cb)  # keep the trampoline alive as long as the world
        self._ck(self._L.sph_fluid_push_host_force(self._w, fluid, cb, None))

    def push_host_force2(self, fluid, solve, contacts=True, boundaries=True):
        """NonPressureForce::solve with its full argument list (nonpressure_force.rs:15-27).  solve(ctx) gets an object with
        dt, inv_dt, kernel_radius, particle_radius, fluid, fluid_index, density0, positions, velocities, densities,
        volumes, accelerations (add in place) and — on request — fluid_fluid_contacts / fluid_boundaries_contacts
        (ContactsView) and boundaries (list of dicts with positions / velocities / volumes)."""
        import types

        def tramp(_user, cp):
            c = cp.contents
            n = c.n
            ctx = types.SimpleNamespace(dt=c.dt, inv_dt=c.inv_dt, kernel_radius=c.kernel_radius, particle_radius=c.particle_radius,
                                        fluid=c.fluid, fluid_index=c.fluid_index, density0=c.density0,
                                        positions=_view(c.positions_xyz, (n, 3)), velocities=_view(c.velocities_xyz, (n, 3)),
                                        densities=_view(c.densities, (n,)), volumes=_view(c.volumes, (n,)) if c.volumes else None,
                                        accelerations=_view(c.accelerations_xyz, (n, 3)),
                                        fluid_fluid_contacts=None, fluid_boundaries_contacts=None, boundaries=None)
            if c.ff_offsets:
                off = _view(c.ff_offsets, (n + 1,), np.uint32)
                m = int(off[-1]) if n else 0
                ctx.fluid_fluid_contacts = ContactsView(off, _view(c.ff_j, (m,), np.uint32), _view(c.ff_j_model, (m,), np.uint32),
                                                        _view(c.ff_weight, (m,)), _view(c.ff_gradient_xyz, (m, 3)))
                off = _view(c.fb_offsets, (n + 1,), np.uint32)
                m = int(off[-1]) if n else 0
                ctx.fluid_boundaries_contacts = ContactsView(off, _view(c.fb_j, (m,), np.uint32), _view(c.fb_j_model, (m,), np.uint32),
                                                             _view(c.fb_weight, (m,)), _view(c.fb_gradient_xyz, (m, 3)))
            if c.boundaries:
                ctx.boundaries = [dict(positions=_view(c.boundaries[b].positions_xyz, (c.boundaries[b].n, 3)),
                                       velocities=_view(c.boundaries[b].velocities_xyz, (c.boundaries[b].n, 3)),
                                       volumes=_view(c.boundaries[b].volumes, (c.boundaries[b].n,))) for b in range(c.n_boundaries)]
            solve(ctx)

        cb = _lib.HOST_FORCE_FN2(tramp)
        self._callbacks.append(cb)
        self._ck(self._L.sph_fluid_push_host_force2(self._w, fluid, cb, None, (1 if contacts else 0) | (2 if boundaries else 0)))

    def remove_fluid(self, fluid):
        """LiquidWorld::remove_fluid liquid_world.rs:171-173"""
        self._ck(self._L.sph_fluid_remove(self._w, fluid))

    def remove_boundary(self, b):
        """LiquidWorld::remove_boundary liquid_world.rs:176-178"""
        self._ck(self._L.sph_boundary_remove(self._w, b))
        self._nb.pop(b, None)

    def set_boundary_particles(self, b, positions, velocities=None):
        """Replace a boundary's whole particle set (a coupled collider re-samples it every step, fluids_pipeline.rs:175-245)."""
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        self._ck(self._L.sph_boundary_set_particles(self._w, b, _fp(p), _fp(v), len(p)))
        self._nb[b] = len(p)

    def step_with_coupling(self, dt, gravity, coupling):
        """LiquidWorld::step_with_coupling liquid_world.rs:67-158 with a CouplingManager (coupling_manager.rs:9-28)."""
        g = np.asarray(gravity, np.float32)
        upd = _lib.COUPLING_UPDATE_FN(lambda _u, _w, dt_, inv_dt, h, r: coupling.update_boundaries(self, dt_, inv_dt, h, r))
        tr = _lib.COUPLING_TRANSMIT_FN(lambda _u, _w, dt_, inv_dt: coupling.transmit_forces(self, dt_, inv_dt))
        cm = _lib.CouplingManagerC(upd, tr, None)
        self._ck(self._L.sph_world_step_with_coupling(self._w, dt, _fp(g), C.byref(cm)))

    # -- collider coupling on the device (ColliderCouplingSet, fluids_pipeline.rs:72-287) ------------------------
    def register_coupling(self, boundary, sampling):
        """ColliderCouplingSet::register_coupling (fluids_pipeline.rs:98-114): couples `boundary` to a new collider and
        returns the collider's handle.  The engine owns the boundary's particles from then on."""
        pts = getattr(sampling, "points", np.zeros((0, 3), np.float32))
        if sampling.kind == DynamicContactSampling.kind and getattr(getattr(sampling, "shape", None), "kind", None) == HEIGHTFIELD:
            h = C.c_uint32()
            self._ck(self._L.sph_collider_register_heightfield(self._w, boundary, C.byref(heightfield_c(sampling.shape)), C.byref(h)))
            self._nb.pop(boundary, None)
            return h.value
        sh = None
        if getattr(sampling, "shape", None) is not None:
            sh = _lib.Shape()
            sh.kind = sampling.shape.kind
            for i, x in enumerate(sampling.shape.params):
                sh.p[i] = x
        h = C.c_uint32()
        self._ck(self._L.sph_collider_register(self._w, boundary, sampling.kind, C.byref(sh) if sh is not None else None, _fp(pts),
                                               len(pts), C.byref(h)))
        if sampling.kind == DynamicContactSampling.kind:
            self._nb.pop(boundary, None)  # resampled every step: its size comes from sph_boundary_count
        else:
            self._nb[boundary] = len(pts)
        return h.value

    def set_collider_state(self, collider, translation=(0.0, 0.0, 0.0), rotation=None, body=BODY_NONE, linvel=(0.0, 0.0, 0.0),
                           angvel=(0.0, 0.0, 0.0), world_com=(0.0, 0.0, 0.0)):
        """The collider's pose (world = rotation @ local + translation, rotation 3x3) and its body for the next steps;
        a body's velocity at p is linvel + angvel x (p - world_com)."""
        s = _lib.ColliderState()
        s.translation[:] = [float(x) for x in translation]
        s.rotation_rowmajor[:] = [float(x) for x in (np.eye(3) if rotation is None else np.asarray(rotation)).reshape(9)]
        s.body = body
        s.linvel[:] = [float(x) for x in linvel]
        s.angvel[:] = [float(x) for x in angvel]
        s.world_com[:] = [float(x) for x in world_com]
        self._ck(self._L.sph_collider_set_state(self._w, collider, C.byref(s)))

    def collider_impulse(self, collider):
        """(linear, angular) impulse the fluid applied to the collider's body in the last step (transmit_forces,
        fluids_pipeline.rs:263-287)."""
        lin, ang = np.zeros(3, np.float32), np.zeros(3, np.float32)
        self._ck(self._L.sph_collider_read_impulse(self._w, collider, _fp(lin), _fp(ang)))
        return lin, ang

    def unregister_coupling(self, collider):
        """ColliderCouplingSet::unregister_coupling (fluids_pipeline.rs:119-122): the boundary stays."""
        self._ck(self._L.sph_collider_unregister(self._w, collider))

    def read_boundary_particles(self, b):
        """boundary.positions / velocities (boundary.rs:13-15) in original index order."""
        n = C.c_size_t()
        self._ck(self._L.sph_boundary_read(self._w, b, None, None, 0, C.byref(n)))
        p, v = np.empty((n.value, 3), np.float32), np.empty((n.value, 3), np.float32)
        self._ck(self._L.sph_boundary_read(self._w, b, _fp(p), _fp(v), n.value, C.byref(n)))
        return p, v

    def particles_intersecting_shape(self, shape, translation=(0.0, 0.0, 0.0), rotation=None):
        """liquid_world.rs:246-281 for Ball / Cuboid / Capsule / Cylinder / Cone / sampling.HeightField under the isometry (rotation 3x3
        row-major, translation)."""
        if shape.kind == HEIGHTFIELD:
            sh = heightfield_c(shape)
            query = self._L.sph_world_particles_in_heightfield
        else:
            sh = _lib.Shape()
            sh.kind = shape.kind
            for i, x in enumerate(shape.params):
                sh.p[i] = x
            query = self._L.sph_world_particles_in_shape
        t = np.ascontiguousarray(translation, np.float32)
        R = None if rotation is None else np.ascontiguousarray(rotation, np.float32).reshape(9)
        n = C.c_size_t(0)
        u32p = C.POINTER(C.c_uint32)
        cap = 1024
        while True:
            k = np.empty(cap, np.uint32)
            h = np.empty(cap, np.uint32)
            i = np.empty(cap, np.uint32)
            self._ck(query(self._w, C.byref(sh), _fp(t), _fp(R), k.ctypes.data_as(u32p), h.ctypes.data_as(u32p), i.ctypes.data_as(u32p), cap,
                           C.byref(n)))
            if n.value <= cap:
                return k[:n.value], h[:n.value], i[:n.value]
            cap = n.value

    # -- particle sinks and sources (faucet3.rs:69-105, include/sph.h, DESIGN.md section 14) ------------------------
    def add_sink(self, fluid, lo, hi, outside=False):
        """Every step, removes the particles of `fluid` in the box lo <= x < hi (outside=True: every particle not in it) at the
        start of the step, on the device.  Returns the sink's handle."""
        d = _lib.SinkDesc()
        d.lo[:] = [float(x) for x in np.asarray(lo, np.float32)]
        d.hi[:] = [float(x) for x in np.asarray(hi, np.float32)]
        d.outside = int(outside)
        h = C.c_uint32()
        self._ck(self._L.sph_fluid_add_sink(self._w, fluid, C.byref(d), C.byref(h)))
        return h.value

    def add_source(self, fluid, positions, velocities=None, interval=1):
        """Appends the template (positions, velocities=None: zero) to `fluid` on the first step and every interval-th step
        after it, as append_particles would.  Returns the source's handle."""
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        if v is not None and len(v) != len(p):
            raise ValueError("add_source: %d velocities for %d positions" % (len(v), len(p)))
        h = C.c_uint32()
        self._ck(self._L.sph_fluid_add_source(self._w, fluid, _fp(p), _fp(v), 0 if p is None else len(p), int(interval), C.byref(h)))
        return h.value

    def remove_sink(self, sink):
        self._ck(self._L.sph_sink_remove(self._w, sink))

    def remove_source(self, source):
        self._ck(self._L.sph_source_remove(self._w, source))

    def step_edits(self, fluid):
        """(removed, emitted): the particles of `fluid` the last step's sinks removed and its sources emitted."""
        r, e = C.c_uint32(), C.c_uint32()
        self._ck(self._L.sph_fluid_read_step_edits(self._w, fluid, C.byref(r), C.byref(e)))
        return r.value, e.value

    # -- fluid surface meshes (include/sph.h, DESIGN.md section 15) -------------------------------------------------
    def extract_surface(self, iso=0.6, spacing=None, fluids=None, box=None, normals=True, anisotropy=None):
        """Samples phi = sum_j V_j W(|x - x_j|) of `fluids` (None: all) on a lattice of `spacing` (None: the particle radius)
        and polygonises phi = iso on the device.  box=None meshes the fluids' AABB grown by h, where every surface closes; a
        box (lo, hi) clips the lattice, and surfaces are open where it cuts them.  anisotropy=None keeps the spherical
        kernels; a SurfaceAnisotropy gives every particle a smoothed centre and an ellipsoidal kernel (include/sph.h
        sph_world_extract_surface_anisotropic), whose rows surface_ellipsoids reads.  Returns (n_vertices, n_triangles); the
        mesh stays on the device until the next extraction."""
        d = _lib.SurfaceDesc()
        d.iso = float(iso)
        d.spacing = float(self.particle_radius if spacing is None else spacing)
        if box is None:
            d.lo[:], d.hi[:] = [1.0, 1.0, 1.0], [0.0, 0.0, 0.0]
        else:
            d.lo[:] = [float(x) for x in np.asarray(box[0], np.float32)]
            d.hi[:] = [float(x) for x in np.asarray(box[1], np.float32)]
        d.normals = int(bool(normals))
        hs = np.ascontiguousarray(np.asarray([] if fluids is None else list(fluids), np.uint32))
        nv, nt = C.c_size_t(), C.c_size_t()
        hp = hs.ctypes.data_as(C.POINTER(C.c_uint32))
        if anisotropy is None:
            self._ck(self._L.sph_world_extract_surface(self._w, hp, len(hs), C.byref(d), C.byref(nv), C.byref(nt)))
        else:
            a = anisotropy._c()
            self._ck(self._L.sph_world_extract_surface_anisotropic(self._w, hp, len(hs), C.byref(d), C.byref(a), C.byref(nv), C.byref(nt)))
        self._surface_normals = bool(normals)
        self._surface_spacing = np.float32(d.spacing)
        self._surface_counts = (nv.value, nt.value)
        return nv.value, nt.value

    def read_surface(self, normals=None):
        """(vertices[nv, 3], triangles[nt, 3], normals[nv, 3] or None) of the last extraction."""
        nv, nt = getattr(self, "_surface_counts", (0, 0))
        if normals is None:
            normals = getattr(self, "_surface_normals", False)
        v = np.empty((nv, 3), np.float32)
        t = np.empty((nt, 3), np.uint32)
        n = np.empty((nv, 3), np.float32) if normals else None
        self._ck(self._L.sph_world_read_surface(self._w, _fp(v), _fp(n) if n is not None else None, nv,
                                                t.ctypes.data_as(C.POINTER(C.c_uint32)), nt))
        return v, t, n

    def surface_mesh(self, iso=0.6, spacing=None, fluids=None, box=None, normals=True, anisotropy=None):
        """extract_surface then read_surface: (vertices[nv, 3] f32, triangles[nt, 3] u32, normals[nv, 3] f32 or None).
        Triangles wind counter-clockwise seen from outside; see include/sph.h for the lattice and the ordering."""
        self.extract_surface(iso, spacing, fluids, box, normals, anisotropy)
        return self.read_surface(normals)

    def surface_ellipsoids(self, fluid):
        """(centres[n, 3] f32, axes[n, 3, 4] f32) of the last extraction for `fluid`, in its particle order: axes[i, k] =
        (e_k, a_k), a_1 >= a_2 >= a_3.  n = 0 after an isotropic extraction or when the fluid was not selected."""
        n = C.c_size_t()
        self._ck(self._L.sph_world_read_surface_ellipsoids(self._w, fluid, None, None, 0, C.byref(n)))
        c, a = np.empty((n.value, 3), np.float32), np.empty((n.value, 3, 4), np.float32)
        self._ck(self._L.sph_world_read_surface_ellipsoids(self._w, fluid, _fp(c), _fp(a), n.value, C.byref(n)))
        return c, a

    def map_surface_ellipsoids(self, fluid):
        """Device views (no host copy) of surface_ellipsoids(fluid)'s (centres[n, 3], axes[n, 3, 4]) as objects with
        __cuda_array_interface__; valid until the next extraction."""
        cp, ap, n = C.POINTER(C.c_float)(), C.POINTER(C.c_float)(), C.c_size_t()
        self._ck(self._L.sph_world_map_surface_ellipsoids(self._w, fluid, C.byref(cp), C.byref(ap), C.byref(n)))

        def view(ptr, shape):
            addr = C.cast(ptr, C.c_void_p).value or 0

            class _View:
                __cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (addr, False), "version": 2, "strides": None}
            return _View()
        return view(cp, (n.value, 3)), view(ap, (n.value, 3, 4))

    def surface_field(self):
        """(phi[nz, ny, nx], origin[3], spacing) of the last extraction's lattice."""
        o = np.zeros(3, np.float32)
        dims = (C.c_uint32 * 3)()
        self._ck(self._L.sph_world_read_surface_field(self._w, None, 0, _fp(o), dims))
        nx, ny, nz = int(dims[0]), int(dims[1]), int(dims[2])
        phi = np.empty((nz, ny, nx), np.float32)
        self._ck(self._L.sph_world_read_surface_field(self._w, _fp(phi), phi.size, _fp(o), dims))
        return phi, o, getattr(self, "_surface_spacing", np.float32(0.0))

    def map_surface(self):
        """Device views (no host copy) of the last extraction's (vertices[nv, 3], triangles[nt, 3], normals[nv, 3] or None) as
        objects with __cuda_array_interface__; valid until the next extraction."""
        nv, nt = getattr(self, "_surface_counts", (0, 0))
        vp, np_, tp = C.POINTER(C.c_float)(), C.POINTER(C.c_float)(), C.POINTER(C.c_uint32)()
        self._ck(self._L.sph_world_map_surface(self._w, C.byref(vp), C.byref(np_), C.byref(tp)))

        def view(ptr, shape, typestr):
            addr = C.cast(ptr, C.c_void_p).value or 0

            class _View:
                __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (addr, False), "version": 2, "strides": None}
            return _View()
        normals = view(np_, (nv, 3), "<f4") if C.cast(np_, C.c_void_p).value else None
        return view(vp, (nv, 3), "<f4"), view(tp, (nt, 3), "<u4"), normals

    # -- diffuse particles: spray, foam and air bubbles (include/sph.h, DESIGN.md section 16) -------------------------
    def diffuse_desc(self, **desc):
        """sph_diffuse_desc_default with `desc`'s fields replaced (lo / hi as 3-sequences)."""
        d = _lib.DiffuseDesc()
        self._L.sph_diffuse_desc_default(C.byref(d))
        for k, v in desc.items():
            if k in ("lo", "hi"):
                getattr(d, k)[:] = [float(x) for x in np.asarray(v, np.float32)]
            elif not hasattr(d, k):
                raise TypeError("unknown diffuse field %r" % k)
            else:
                setattr(d, k, v)
        return d

    def update_diffuse(self, dt, gravity=(0.0, -9.81, 0.0), fluids=None, **desc):
        """Advances the world's diffuse set by one frame of length dt from `fluids` (None: all), on the device.  desc fields
        (include/sph.h sph_diffuse_desc) override the defaults.  Returns the update's stats as a dict."""
        d = self.diffuse_desc(**desc)
        hs = np.ascontiguousarray(np.asarray([] if fluids is None else list(fluids), np.uint32))
        g = np.ascontiguousarray(np.asarray(gravity, np.float32).reshape(3))
        st = _lib.DiffuseStats()
        self._ck(self._L.sph_world_update_diffuse(self._w, hs.ctypes.data_as(C.POINTER(C.c_uint32)), len(hs), C.byref(d), float(dt), _fp(g),
                                                  C.byref(st)))
        return {k: int(getattr(st, k)) for k, _ in _lib.DiffuseStats._fields_}

    def diffuse_particles(self):
        """(positions[n, 3] f32, velocities[n, 3] f32, kinds[n] u8 (0 spray, 1 foam, 2 bubble), lives[n] f32) in order."""
        n = C.c_size_t()
        self._ck(self._L.sph_world_read_diffuse(self._w, None, None, None, None, 0, C.byref(n)))
        p, v = np.empty((n.value, 3), np.float32), np.empty((n.value, 3), np.float32)
        k, life = np.empty(n.value, np.uint8), np.empty(n.value, np.float32)
        self._ck(self._L.sph_world_read_diffuse(self._w, _fp(p), _fp(v), k.ctypes.data_as(C.POINTER(C.c_uint8)), _fp(life), n.value, C.byref(n)))
        return p, v, k, life

    def map_diffuse(self):
        """Device views (no host copy) of (positions[n, 3], velocities[n, 3], kinds[n], lives[n]) as objects with
        __cuda_array_interface__; valid until the next update or clear."""
        ptrs = [C.POINTER(C.c_float)(), C.POINTER(C.c_float)(), C.POINTER(C.c_uint8)(), C.POINTER(C.c_float)()]
        n = C.c_size_t()
        self._ck(self._L.sph_world_map_diffuse(self._w, *[C.byref(x) for x in ptrs], C.byref(n)))

        def view(ptr, shape, typestr):
            addr = C.cast(ptr, C.c_void_p).value or 0

            class _View:
                __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (addr, False), "version": 2, "strides": None}
            return _View()
        m = n.value
        return view(ptrs[0], (m, 3), "<f4"), view(ptrs[1], (m, 3), "<f4"), view(ptrs[2], (m,), "|u1"), view(ptrs[3], (m,), "<f4")

    def clear_diffuse(self):
        """Empties the diffuse set."""
        self._ck(self._L.sph_world_clear_diffuse(self._w))

    # -- snapshot / restore and zero-copy views (include/sph.h) ---------------------------------------------
    def snapshot(self):
        """Everything the solver carries across steps (vc, dt lag, IISPH pressures, Becker rest pose, ids) as bytes."""
        n = C.c_size_t()
        self._ck(self._L.sph_world_snapshot_size(self._w, C.byref(n)))
        buf = (C.c_char * n.value)()
        wr = C.c_size_t()
        self._ck(self._L.sph_world_snapshot_save(self._w, buf, n.value, C.byref(wr)))
        return bytes(buf[:wr.value])

    def restore(self, blob):
        buf = C.create_string_buffer(blob, len(blob))
        self._ck(self._L.sph_world_snapshot_load(self._w, buf, len(blob)))

    def map_positions(self, fluid, velocities=False):
        """Device view (no host copy) of fluid.positions in ORIGINAL index order: an object with __cuda_array_interface__
        (torch.as_tensor(view, device='cuda') / cupy.asarray(view)); valid until the next call on this world."""
        ptr = C.POINTER(C.c_float)()
        n = C.c_size_t()
        fn = self._L.sph_fluid_map_velocities if velocities else self._L.sph_fluid_map_positions
        self._ck(fn(self._w, fluid, C.byref(ptr), C.byref(n)))
        addr = C.cast(ptr, C.c_void_p).value or 0

        class _View:
            __cuda_array_interface__ = {"shape": (n.value, 3), "typestr": "<f4", "data": (addr, False), "version": 2, "strides": None}
        return _View()

    def add_boundary(self, boundary_or_positions, velocities=None, memberships=1, filter=0xFFFFFFFF,
                     want_forces=False):
        if isinstance(boundary_or_positions, Boundary):
            b = boundary_or_positions
            p, velocities, want_forces = b.positions, b.velocities, b.want_forces
            memberships, filter = b.interaction_groups.memberships, b.interaction_groups.filter
        else:
            p = boundary_or_positions
        p = _f32(p, (-1, 3))
        v = _f32(velocities, (-1, 3))
        h = C.c_uint32()
        self._ck(self._L.sph_boundary_add(self._w, _fp(p), _fp(v), len(p), memberships, filter, int(want_forces),
                                          C.byref(h)))
        self._nb[h.value] = len(p)
        return h.value

    def step(self, dt, gravity=(0.0, -9.81, 0.0)):
        g = np.asarray(gravity, np.float32)
        self._ck(self._L.sph_world_step(self._w, dt, _fp(g)))

    def step_many(self, dt, n_steps, gravity=(0.0, -9.81, 0.0)):
        """n_steps calls of step(dt, gravity), steps 2..n_steps as one CUDA graph (include/sph.h sph_world_step_many).
        Returns the number of steps done; raises SphError as step does, with the steps done before the failing one in its
        steps_done attribute."""
        g = np.asarray(gravity, np.float32)
        done = C.c_uint32()
        st = self._L.sph_world_step_many(self._w, dt, _fp(g), n_steps, C.byref(done))
        if st != 0:
            e = SphError(st, self._L.sph_last_error(self._w).decode())
            e.steps_done = done.value
            raise e
        return done.value

    def step_records(self):
        """One dict per step of the last step / step_many call (include/sph.h sph_step_record)."""
        n = C.c_size_t()
        self._ck(self._L.sph_world_read_step_records(self._w, None, 0, C.byref(n)))
        out = (_lib.StepRecord * max(n.value, 1))()
        self._ck(self._L.sph_world_read_step_records(self._w, out, n.value, C.byref(n)))
        return [{f: getattr(out[i], f) for f, _ in _lib.StepRecord._fields_} for i in range(n.value)]

    def set_substepping(self, cfl_coeff=0.4, min_substeps=1, max_substeps=10):
        """CFL-bounded substeps inside each step (include/sph.h sph_world_set_substepping); the defaults are the reference
        TimestepManager's (timestep_manager.rs:21-31).  cfl_coeff=0 turns substepping off."""
        self._ck(self._L.sph_world_set_substepping(self._w, cfl_coeff, min_substeps, max_substeps))

    def substeps(self):
        """The lengths of the last step's substeps, in order, as float32 (empty when the step ran no solver)."""
        n = C.c_size_t()
        self._ck(self._L.sph_world_read_substeps(self._w, None, 0, C.byref(n)))
        out = np.empty(n.value, np.float32)
        self._ck(self._L.sph_world_read_substeps(self._w, _fp(out), n.value, C.byref(n)))
        return out

    # -- particle access (fluids_mut() edits, fluid.rs / liquid_world.rs:181-198) -------------------
    def num_particles(self, fluid):
        n = C.c_size_t()
        self._ck(self._L.sph_fluid_count(self._w, fluid, C.byref(n)))
        return n.value

    def read_fluid(self, fluid, positions=None, velocities=None):
        """Returns (positions, velocities) in ORIGINAL index order; optional preallocated outputs."""
        n = self.num_particles(fluid)
        p = np.empty((n, 3), np.float32) if positions is None else positions
        v = np.empty((n, 3), np.float32) if velocities is None else velocities
        m = C.c_size_t()
        self._ck(self._L.sph_fluid_read(self._w, fluid, _fp(p), _fp(v), n, C.byref(m)))
        return p, v

    def write_fluid(self, fluid, positions=None, velocities=None):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        n = len(p) if p is not None else len(v)
        self._ck(self._L.sph_fluid_write(self._w, fluid, _fp(p), _fp(v), n))

    def append_particles(self, fluid, positions, velocities=None):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        self._ck(self._L.sph_fluid_append(self._w, fluid, _fp(p), _fp(v), len(p)))

    def delete_particles(self, fluid, mask):
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        self._ck(self._L.sph_fluid_delete(self._w, fluid, m.ctypes.data_as(C.POINTER(C.c_uint8)), len(m)))

    def write_boundary(self, b, positions=None, velocities=None):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        n = len(p) if p is not None else len(v) if v is not None else self._boundary_count(b)  # the library refuses a wrong length
        self._ck(self._L.sph_boundary_write(self._w, b, _fp(p), _fp(v), n))

    def _boundary_count(self, b):
        if b in self._nb:
            return self._nb[b]
        n = C.c_size_t()
        self._ck(self._L.sph_boundary_count(self._w, b, C.byref(n)))
        return n.value

    def read_boundary(self, b):
        n = self._boundary_count(b)
        vol = np.empty(n, np.float32)
        f = np.zeros((n, 3), np.float32)
        self._ck(self._L.sph_boundary_read_volumes(self._w, b, _fp(vol), n))
        self._ck(self._L.sph_boundary_read_forces(self._w, b, _fp(f), n))
        return vol, f

    def particles_intersecting_aabb(self, mins, maxs):
        """liquid_world.rs:211-243 -> (kinds, handles, indices) uint32 arrays sorted by (kind, handle, index);
        kind 0 = fluid particle, 1 = boundary particle."""
        lo = np.ascontiguousarray(mins, np.float32)
        hi = np.ascontiguousarray(maxs, np.float32)
        n = C.c_size_t(0)
        u32p = C.POINTER(C.c_uint32)
        cap = 1024
        while True:
            k = np.empty(cap, np.uint32)
            h = np.empty(cap, np.uint32)
            i = np.empty(cap, np.uint32)
            self._ck(self._L.sph_world_particles_in_aabb(self._w, _fp(lo), _fp(hi), k.ctypes.data_as(u32p), h.ctypes.data_as(u32p),
                                                         i.ctypes.data_as(u32p), cap, C.byref(n)))
            if n.value <= cap:
                return k[:n.value], h[:n.value], i[:n.value]
            cap = n.value

    # -- particle ids and multi-GPU slabs (include/sph.h "Multi-GPU") --------------------------------------
    def set_ids(self, fluid, ids):
        a = np.ascontiguousarray(ids, dtype=np.uint32)
        self._ck(self._L.sph_fluid_set_ids(self._w, fluid, a.ctypes.data_as(C.POINTER(C.c_uint32)), len(a)))

    def read_ids(self, fluid):
        n = self.num_particles(fluid)
        a = np.empty(n, np.uint32)
        self._ck(self._L.sph_fluid_read_ids(self._w, fluid, a.ctypes.data_as(C.POINTER(C.c_uint32)), n))
        return a

    def replace_particles(self, fluid, positions, velocities=None, velocity_changes=None, ids=None):
        """Replace a fluid's whole particle set (slab re-balancing: particles change rank wholesale)."""
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        c = _f32(velocity_changes, (-1, 3))
        i = None if ids is None else np.ascontiguousarray(ids, dtype=np.uint32)
        ip = None if i is None else i.ctypes.data_as(C.POINTER(C.c_uint32))
        self._ck(self._L.sph_fluid_replace_particles(self._w, fluid, _fp(p), _fp(v), _fp(c), ip, len(p)))

    def set_slab(self, cell_lo, cell_hi):
        self._ck(self._L.sph_world_set_slab(self._w, int(cell_lo), int(cell_hi)))

    def init_slab(self, unique_id, rank, nranks, cell_lo, cell_hi):
        """Join the slab decomposition: `unique_id` is the 128-byte NCCL id rank 0 got from nccl_unique_id()."""
        self._ck(self._L.sph_world_create_nccl(self._w, bytes(unique_id), rank, nranks))
        self._ck(self._L.sph_world_set_slab(self._w, int(cell_lo), int(cell_hi)))

    # -- parity / bench aids -----------------------------------------------------------------------
    def force_iterations(self, n_div=-1, n_press=-1):
        self._ck(self._L.sph_world_force_iterations(self._w, n_div, n_press))

    def stats(self):
        s = StepStats()
        self._ck(self._L.sph_world_stats(self._w, C.byref(s)))
        out = {}
        for name, _ in StepStats._fields_:
            v = getattr(s, name)
            out[name] = list(v) if name == "grid_dims" else v
        return out

    def debug(self, fluid, what):
        code = DBG[what] if isinstance(what, str) else what
        n = self.num_particles(fluid)
        out = np.zeros((n, WIDTH[code]) if code in WIDTH else (n,), np.float32)
        self._ck(self._L.sph_debug_read(self._w, fluid, code, _fp(out), n))
        return out
