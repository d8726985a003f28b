"""ctypes binding of oracle/liboracle.so — the CPU restatement of salva3d's step path.

TEST INFRASTRUCTURE ONLY (parity checker + timed CPU baseline).  PARITY UNPINNED by the
reference (no golden vectors exist upstream); pinned by tests/test_oracle_*.py instead.
The class mirrors the product's host mirror (salva_b200.liquid_world) closely enough that
parity tests drive both with the same scene description.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class OrcDesc(C.Structure):
    _fields_ = [("solver", C.c_int32), ("particle_radius", C.c_float), ("smoothing_factor", C.c_float),
                ("min_pressure_iter", C.c_uint32), ("max_pressure_iter", C.c_uint32),
                ("max_density_error", C.c_float),
                ("min_divergence_iter", C.c_uint32), ("max_divergence_iter", C.c_uint32),
                ("max_divergence_error", C.c_float), ("omega", C.c_float),
                ("sort_contacts", C.c_int32), ("num_threads", C.c_int32)]


class OrcStats(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("step_ms", "grid_ms", "neighbors_ms", "density_ms", "divergence_ms",
                                         "nonpressure_ms", "pressure_ms", "integrate_ms")] + \
               [(n, C.c_uint32) for n in ("n_divergence_iter", "n_pressure_iter", "n_divergence_eval",
                                          "n_pressure_eval")] + \
               [("last_divergence_error", C.c_float), ("last_density_error", C.c_float),
                ("n_contacts", C.c_uint64), ("threads", C.c_int32)]


HOST_FORCE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_size_t, C.POINTER(C.c_float), C.POINTER(C.c_float),
                            C.POINTER(C.c_float), C.POINTER(C.c_float))


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-B", "liboracle.so"], check=True, capture_output=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        fp, u8p, vp = C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.c_void_p
        L.orc_world_create.restype = vp
        L.orc_world_create.argtypes = [C.POINTER(OrcDesc)]
        L.orc_world_destroy.argtypes = [vp]
        L.orc_fluid_add.argtypes = [vp, fp, fp, fp, C.c_size_t, C.c_float, C.c_uint32, C.c_uint32]
        L.orc_fluid_push_force.argtypes = [vp, C.c_uint32, C.c_int, fp]
        u32p = C.POINTER(C.c_uint32)
        L.orc_particles_in_aabb.argtypes = [vp, fp, fp, u32p, u32p, u32p, C.c_size_t]
        L.orc_particles_in_aabb.restype = C.c_size_t
        L.orc_fluid_append.argtypes = [vp, C.c_uint32, fp, fp, C.c_size_t]
        L.orc_fluid_push_host_force.argtypes = [vp, C.c_uint32, HOST_FORCE_FN, vp]
        L.orc_fluid_delete.argtypes = [vp, C.c_uint32, u8p, C.c_size_t]
        L.orc_fluid_write.argtypes = [vp, C.c_uint32, fp, fp, C.c_size_t]
        L.orc_fluid_count.restype = C.c_size_t
        L.orc_fluid_count.argtypes = [vp, C.c_uint32]
        L.orc_fluid_read.argtypes = [vp, C.c_uint32, fp, fp]
        L.orc_boundary_add.argtypes = [vp, fp, fp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int]
        L.orc_boundary_write.argtypes = [vp, C.c_uint32, fp, fp, C.c_size_t]
        L.orc_boundary_read.argtypes = [vp, C.c_uint32, fp, fp]
        L.orc_world_step.argtypes = [vp, C.c_float, fp]
        L.orc_world_force_iterations.argtypes = [vp, C.c_int, C.c_int]
        L.orc_world_stats.argtypes = [vp, C.POINTER(OrcStats)]
        L.orc_debug_read.argtypes = [vp, C.c_uint32, C.c_int, fp]
        L.orc_last_error.restype = C.c_char_p
        L.orc_last_error.argtypes = [vp]
        for n in ("orc_kernel_w", "orc_kernel_dw", "orc_cohesion_kernel", "orc_adhesion_kernel"):
            getattr(L, n).restype = C.c_float
            getattr(L, n).argtypes = [C.c_float, C.c_float]
        L.orc_world_set_kernels.argtypes = [vp, C.c_int, C.c_int]
        for n in ("orc_kernel_w_kind", "orc_kernel_dw_kind"):
            getattr(L, n).restype = C.c_float
            getattr(L, n).argtypes = [C.c_int, C.c_float, C.c_float]
        L.orc_max_threads.restype = C.c_int
        _LIB = L
    return _LIB


def _fp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def _f32(a, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float32)
    if shape is not None:
        a = a.reshape(shape)
    return a


DBG = dict(density=0, alpha=1, divergence=2, predicted_density=3, velocity_change=4, num_fluid_contacts=5,
           num_boundary_contacts=6, pressure=7, acceleration=8, dii=9, aii=10, dij_pjl=11, he2014_color=12, he2014_gradc=13,
           visc_beta=14, visc_target=15, el_volume0=16, el_rotation=17, el_grad_tr=18, el_stress=19)
# floats per particle of the selectors that are not scalars (include/sph.h)
WIDTH = {4: 3, 8: 3, 9: 3, 11: 3, 14: 36, 15: 6, 17: 9, 18: 9, 19: 6}


class OracleWorld:
    """LiquidWorld restatement (liquid_world.rs:17-158) on the CPU oracle."""

    def __init__(self, particle_radius, smoothing_factor=2.0, solver=0, min_pressure_iter=1, max_pressure_iter=50,
                 max_density_error=0.05, min_divergence_iter=1, max_divergence_iter=50, max_divergence_error=0.1,
                 omega=0.5, sort_contacts=True, num_threads=None, kernel_density=0, kernel_gradient=0):
        self._L = lib()
        if num_threads is None:  # small test scenes: a handful of threads (128 spinning OpenMP threads are far slower)
            num_threads = min(8, os.cpu_count() or 1)
        d = OrcDesc(solver, particle_radius, smoothing_factor, min_pressure_iter, max_pressure_iter,
                    max_density_error, min_divergence_iter, max_divergence_iter, max_divergence_error, omega,
                    int(sort_contacts), num_threads)
        self._w = self._L.orc_world_create(C.byref(d))
        if kernel_density or kernel_gradient:  # DFSPHSolver<KernelDensity, KernelGradient> dfsph_solver.rs:17-20
            self._L.orc_world_set_kernels(self._w, kernel_density, kernel_gradient)
        self.h = np.float32(particle_radius) * np.float32(smoothing_factor) * np.float32(2.0)
        self.particle_radius = particle_radius

    def __del__(self):
        if getattr(self, "_w", None):
            self._L.orc_world_destroy(self._w)
            self._w = None

    def add_fluid(self, positions, density0=1000.0, velocities=None, volumes=None, memberships=1,
                  filter=0xFFFFFFFF):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        vol = _f32(volumes)
        return self._L.orc_fluid_add(self._w, _fp(p), _fp(v), _fp(vol), len(p), density0, memberships, filter)

    def push_force(self, fluid, kind, params):
        pr = np.zeros(8, np.float32)
        pr[:len(params)] = params
        assert self._L.orc_fluid_push_force(self._w, fluid, kind, _fp(pr)) == 0

    def particles_intersecting_aabb(self, mins, maxs):
        lo = np.ascontiguousarray(mins, np.float32)
        hi = np.ascontiguousarray(maxs, np.float32)
        u32p = C.POINTER(C.c_uint32)
        cap = 1024
        while True:
            k = np.empty(cap, np.uint32)
            h = np.empty(cap, np.uint32)
            i = np.empty(cap, np.uint32)
            n = self._L.orc_particles_in_aabb(self._w, _fp(lo), _fp(hi), k.ctypes.data_as(u32p), h.ctypes.data_as(u32p),
                                              i.ctypes.data_as(u32p), cap)
            if n <= cap:
                return k[:n], h[:n], i[:n]
            cap = n

    def push_host_force(self, fluid, solve):
        def tramp(_user, dt, inv_dt, h, n, pos, vel, dens, acc):
            solve(dt, inv_dt, h, np.ctypeslib.as_array(pos, (n, 3)), np.ctypeslib.as_array(vel, (n, 3)),
                  np.ctypeslib.as_array(dens, (n,)), np.ctypeslib.as_array(acc, (n, 3)))
        cb = HOST_FORCE_FN(tramp)
        if not hasattr(self, "_callbacks"):
            self._callbacks = []
        self._callbacks.append(cb)
        assert self._L.orc_fluid_push_host_force(self._w, fluid, cb, None) == 0

    def append_particles(self, fluid, positions, velocities=None):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        assert self._L.orc_fluid_append(self._w, fluid, _fp(p), _fp(v), len(p)) == 0

    def delete_particles(self, fluid, mask):
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        assert self._L.orc_fluid_delete(self._w, fluid, m.ctypes.data_as(C.POINTER(C.c_uint8)), len(m)) == 0

    def write_fluid(self, fluid, positions=None, velocities=None):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        n = len(p) if p is not None else len(v)
        assert self._L.orc_fluid_write(self._w, fluid, _fp(p), _fp(v), n) == 0

    def num_particles(self, fluid):
        return self._L.orc_fluid_count(self._w, fluid)

    def read_fluid(self, fluid):
        n = self.num_particles(fluid)
        p = np.empty((n, 3), np.float32)
        v = np.empty((n, 3), np.float32)
        assert self._L.orc_fluid_read(self._w, fluid, _fp(p), _fp(v)) == 0
        return p, v

    def add_boundary(self, positions, velocities=None, memberships=1, filter=0xFFFFFFFF, want_forces=False):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        b = self._L.orc_boundary_add(self._w, _fp(p), _fp(v), len(p), memberships, filter, int(want_forces))
        if not hasattr(self, "_bn"):
            self._bn = {}
        self._bn[b] = len(p)
        return b

    def write_boundary(self, b, positions=None, velocities=None):
        p = _f32(positions, (-1, 3))
        v = _f32(velocities, (-1, 3))
        assert self._L.orc_boundary_write(self._w, b, _fp(p), _fp(v), self._bn[b]) == 0

    def read_boundary(self, b):
        n = self._bn[b]
        vol = np.empty(n, np.float32)
        f = np.zeros((n, 3), np.float32)
        assert self._L.orc_boundary_read(self._w, b, _fp(vol), _fp(f)) == 0
        return vol, f

    def step(self, dt, gravity=(0.0, -9.81, 0.0)):
        g = np.asarray(gravity, np.float32)
        rc = self._L.orc_world_step(self._w, dt, _fp(g))
        if rc != 0:
            raise RuntimeError("oracle step failed: %s" % self._L.orc_last_error(self._w).decode())

    def force_iterations(self, n_div=-1, n_press=-1):
        self._L.orc_world_force_iterations(self._w, n_div, n_press)

    def stats(self):
        s = OrcStats()
        self._L.orc_world_stats(self._w, C.byref(s))
        return {n: getattr(s, n) for n, _ in OrcStats._fields_}

    def debug(self, fluid, what):
        code = DBG[what] if isinstance(what, str) else what
        n = self.num_particles(fluid)
        out = np.zeros((n, WIDTH[code]) if code in WIDTH else (n,), np.float32)
        assert self._L.orc_debug_read(self._w, fluid, code, _fp(out)) == 0
        return out
