"""ctypes binding of libsalva_b200.so (the C ABI declared in include/sph.h).

There is no fallback: if the CUDA library is missing or fails to load, importing a world fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SALVA_B200_LIB") or os.path.join(_HERE, "libsalva_b200.so")  # env override: A/B builds
KERNELS_LIB_PATH = os.path.join(_HERE, "libsalva_b200_kernels.so")  # same ABI, solver kernels other than the cubic spline
_LIB = None
_LIBS = {}

SPH_OK = 0
STATUS_NAMES = {0: "SPH_OK", 1: "SPH_ERR_INVALID", 2: "SPH_ERR_CUDA", 3: "SPH_ERR_OOM", 4: "SPH_ERR_NCCL",
                5: "SPH_ERR_ZERO_DENSITY"}


class WorldDesc(C.Structure):
    _fields_ = [("solver", C.c_int32), ("particle_radius", C.c_float), ("smoothing_factor", C.c_float),
                ("min_pressure_iter", C.c_uint32), ("max_pressure_iter", C.c_uint32), ("max_density_error", C.c_float),
                ("min_divergence_iter", C.c_uint32), ("max_divergence_iter", C.c_uint32),
                ("max_divergence_error", C.c_float), ("omega", C.c_float), ("device", C.c_int32),
                ("slab_rank", C.c_int32), ("slab_count", C.c_int32), ("deterministic", C.c_int32),
                ("gather_backend", C.c_int32), ("kernel_density", C.c_int32), ("kernel_gradient", C.c_int32)]


class ForceDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("p", C.c_float * 8)]


class StepStats(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("step_ms", "grid_ms", "neighbors_ms", "density_ms", "divergence_ms",
                                         "nonpressure_ms", "pressure_ms", "integrate_ms", "divergence_eval_ms",
                                         "divergence_update_ms", "predict_density_ms", "pressure_update_ms")] + \
               [(n, C.c_uint32) for n in ("n_divergence_iter", "n_pressure_iter", "n_divergence_eval",
                                          "n_pressure_eval")] + \
               [("last_divergence_error", C.c_float), ("last_density_error", C.c_float),
                ("n_fluid_particles", C.c_uint64), ("n_boundary_particles", C.c_uint64), ("n_contacts", C.c_uint64),
                ("max_neighbors", C.c_uint32), ("grid_dims", C.c_uint32 * 3), ("kernel_launches", C.c_uint64),
                ("n_ghost_particles", C.c_uint32), ("n_migrated", C.c_uint32), ("n_exchanges", C.c_uint32),
                ("n_substeps", C.c_uint32)]


_fp, _u8p, _vp = C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.c_void_p
HOST_FORCE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_size_t, C.POINTER(C.c_float), C.POINTER(C.c_float),
                            C.POINTER(C.c_float), C.POINTER(C.c_float))



class StepRecord(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_divergence_iter", "n_pressure_iter", "n_divergence_eval", "n_pressure_eval")] + \
               [("last_divergence_error", C.c_float), ("last_density_error", C.c_float), ("max_neighbors", C.c_uint32),
                ("on_device", C.c_uint32), ("n_contacts", C.c_uint64)]


class BoundaryView(C.Structure):
    _fields_ = [("n", C.c_size_t), ("positions_xyz", C.POINTER(C.c_float)), ("velocities_xyz", C.POINTER(C.c_float)),
                ("volumes", C.POINTER(C.c_float))]


class HostForceCtx(C.Structure):
    _u32p, _f32p = C.POINTER(C.c_uint32), C.POINTER(C.c_float)
    _fields_ = [("dt", C.c_float), ("inv_dt", C.c_float), ("kernel_radius", C.c_float), ("particle_radius", C.c_float),
                ("fluid", C.c_uint32), ("fluid_index", C.c_uint32), ("density0", C.c_float), ("n", C.c_size_t),
                ("positions_xyz", _f32p), ("velocities_xyz", _f32p), ("densities", _f32p), ("volumes", _f32p),
                ("accelerations_xyz", _f32p),
                ("ff_offsets", _u32p), ("ff_j", _u32p), ("ff_j_model", _u32p), ("ff_weight", _f32p), ("ff_gradient_xyz", _f32p),
                ("fb_offsets", _u32p), ("fb_j", _u32p), ("fb_j_model", _u32p), ("fb_weight", _f32p), ("fb_gradient_xyz", _f32p),
                ("n_boundaries", C.c_size_t), ("boundaries", C.POINTER(BoundaryView))]


class Shape(C.Structure):
    _fields_ = [("kind", C.c_int32), ("p", C.c_float * 4)]


class HeightFieldC(C.Structure):
    _fields_ = [("nrows", C.c_uint32), ("ncols", C.c_uint32), ("heights", C.POINTER(C.c_float)), ("scale", C.c_float * 3)]


class ColliderState(C.Structure):
    _fields_ = [("translation", C.c_float * 3), ("rotation_rowmajor", C.c_float * 9), ("body", C.c_int32),
                ("linvel", C.c_float * 3), ("angvel", C.c_float * 3), ("world_com", C.c_float * 3)]


HOST_FORCE_FN2 = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(HostForceCtx))
COUPLING_UPDATE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float)
COUPLING_TRANSMIT_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_float, C.c_float)


class CouplingManagerC(C.Structure):
    _fields_ = [("update_boundaries", COUPLING_UPDATE_FN), ("transmit_forces", COUPLING_TRANSMIT_FN), ("user", C.c_void_p)]


class SinkDesc(C.Structure):
    _fields_ = [("lo", C.c_float * 3), ("hi", C.c_float * 3), ("outside", C.c_int32)]


class SurfaceDesc(C.Structure):
    _fields_ = [("iso", C.c_float), ("spacing", C.c_float), ("lo", C.c_float * 3), ("hi", C.c_float * 3), ("normals", C.c_int32)]


class SurfaceAnisotropy(C.Structure):
    _fields_ = [("smoothing", C.c_float), ("max_ratio", C.c_float), ("isolated_radius", C.c_float), ("min_neighbours", C.c_uint32)]


class DiffuseDesc(C.Structure):
    _fields_ = [("ta_min", C.c_float), ("ta_max", C.c_float), ("wc_min", C.c_float), ("wc_max", C.c_float), ("k_min", C.c_float),
                ("k_max", C.c_float), ("k_ta", C.c_float), ("k_wc", C.c_float), ("lifetime", C.c_float), ("k_b", C.c_float),
                ("k_d", C.c_float), ("spray_below", C.c_uint32), ("bubble_above", C.c_uint32), ("capacity", C.c_uint32),
                ("seed", C.c_uint32), ("lo", C.c_float * 3), ("hi", C.c_float * 3)]


class DiffuseStats(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ("emitted", "dropped", "expired", "left_box", "spray", "foam", "bubble")]


# every symbol include/sph.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "sph_world_desc_default": (None, [C.POINTER(WorldDesc)]),
    "sph_world_create": (C.c_int, [C.POINTER(WorldDesc), C.POINTER(_vp)]),
    "sph_world_destroy": (None, [_vp]),
    "sph_fluid_add": (C.c_int, [_vp, _fp, _fp, _fp, C.c_size_t, C.c_float, C.c_uint32, C.c_uint32,
                                C.POINTER(C.c_uint32)]),
    "sph_fluid_push_force": (C.c_int, [_vp, C.c_uint32, C.POINTER(ForceDesc)]),
    "sph_world_particles_in_aabb": (C.c_int, [_vp, _fp, _fp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                              C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_fluid_push_host_force": (C.c_int, [_vp, C.c_uint32, HOST_FORCE_FN, _vp]),
    "sph_fluid_append": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t]),
    "sph_fluid_delete": (C.c_int, [_vp, C.c_uint32, _u8p, C.c_size_t]),
    "sph_fluid_write": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t]),
    "sph_fluid_read": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_fluid_count": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_size_t)]),
    "sph_boundary_add": (C.c_int, [_vp, _fp, _fp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int,
                                   C.POINTER(C.c_uint32)]),
    "sph_boundary_write": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t]),
    "sph_boundary_read_forces": (C.c_int, [_vp, C.c_uint32, _fp, C.c_size_t]),
    "sph_boundary_read_volumes": (C.c_int, [_vp, C.c_uint32, _fp, C.c_size_t]),
    "sph_world_step": (C.c_int, [_vp, C.c_float, _fp]),
    "sph_world_step_many": (C.c_int, [_vp, C.c_float, _fp, C.c_uint32, C.POINTER(C.c_uint32)]),
    "sph_world_read_step_records": (C.c_int, [_vp, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_force_iterations": (C.c_int, [_vp, C.c_int32, C.c_int32]),
    "sph_world_set_substepping": (C.c_int, [_vp, C.c_float, C.c_uint32, C.c_uint32]),
    "sph_world_read_substeps": (C.c_int, [_vp, _fp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_stats": (C.c_int, [_vp, C.POINTER(StepStats)]),
    "sph_world_h": (C.c_float, [_vp]),
    "sph_world_particle_radius": (C.c_float, [_vp]),
    "sph_debug_read": (C.c_int, [_vp, C.c_uint32, C.c_int, _fp, C.c_size_t]),
    "sph_last_error": (C.c_char_p, [_vp]),
    "sph_version": (C.c_char_p, []),
    "sph_world_attach_nccl": (C.c_int, [_vp, _vp, C.c_int, C.c_int]),
    "sph_world_create_nccl": (C.c_int, [_vp, C.c_char_p, C.c_int, C.c_int]),
    "sph_world_set_slab": (C.c_int, [_vp, C.c_int32, C.c_int32]),
    "sph_nccl_unique_id": (C.c_int, [C.c_char_p]),
    "sph_fluid_set_ids": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_uint32), C.c_size_t]),
    "sph_fluid_push_host_force2": (C.c_int, [_vp, C.c_uint32, HOST_FORCE_FN2, _vp, C.c_uint32]),
    "sph_fluid_remove": (C.c_int, [_vp, C.c_uint32]),
    "sph_fluid_replace_particles": (C.c_int, [_vp, C.c_uint32, _fp, _fp, _fp, C.POINTER(C.c_uint32), C.c_size_t]),
    "sph_fluid_map_positions": (C.c_int, [_vp, C.c_uint32, C.POINTER(_fp), C.POINTER(C.c_size_t)]),
    "sph_fluid_map_velocities": (C.c_int, [_vp, C.c_uint32, C.POINTER(_fp), C.POINTER(C.c_size_t)]),
    "sph_boundary_remove": (C.c_int, [_vp, C.c_uint32]),
    "sph_boundary_set_particles": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t]),
    "sph_boundary_count": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_size_t)]),
    "sph_world_particles_in_shape": (C.c_int, [_vp, C.POINTER(Shape), _fp, _fp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                               C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_step_with_coupling": (C.c_int, [_vp, C.c_float, _fp, C.POINTER(CouplingManagerC)]),
    "sph_world_snapshot_size": (C.c_int, [_vp, C.POINTER(C.c_size_t)]),
    "sph_world_snapshot_save": (C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_snapshot_load": (C.c_int, [_vp, _vp, C.c_size_t]),
    "sph_fluid_read_ids": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_uint32), C.c_size_t]),
    "sph_collider_register": (C.c_int, [_vp, C.c_uint32, C.c_int32, C.POINTER(Shape), _fp, C.c_size_t, C.POINTER(C.c_uint32)]),
    "sph_collider_set_state": (C.c_int, [_vp, C.c_uint32, C.POINTER(ColliderState)]),
    "sph_collider_read_impulse": (C.c_int, [_vp, C.c_uint32, _fp, _fp]),
    "sph_collider_unregister": (C.c_int, [_vp, C.c_uint32]),
    "sph_boundary_read": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_sample_shape": (C.c_int, [_vp, C.c_int32, C.POINTER(Shape), C.POINTER(HeightFieldC), C.c_float, _fp, C.c_size_t,
                                         C.POINTER(C.c_size_t)]),
    "sph_world_particles_in_heightfield": (C.c_int, [_vp, C.POINTER(HeightFieldC), _fp, _fp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                                     C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_collider_register_heightfield": (C.c_int, [_vp, C.c_uint32, C.POINTER(HeightFieldC), C.POINTER(C.c_uint32)]),
    "sph_fluid_add_sink": (C.c_int, [_vp, C.c_uint32, C.POINTER(SinkDesc), C.POINTER(C.c_uint32)]),
    "sph_sink_remove": (C.c_int, [_vp, C.c_uint32]),
    "sph_fluid_add_source": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t, C.c_uint32, C.POINTER(C.c_uint32)]),
    "sph_source_remove": (C.c_int, [_vp, C.c_uint32]),
    "sph_fluid_read_step_edits": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "sph_world_extract_surface": (C.c_int, [_vp, C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(SurfaceDesc), C.POINTER(C.c_size_t),
                                            C.POINTER(C.c_size_t)]),
    "sph_world_read_surface": (C.c_int, [_vp, _fp, _fp, C.c_size_t, C.POINTER(C.c_uint32), C.c_size_t]),
    "sph_world_map_surface": (C.c_int, [_vp, C.POINTER(_fp), C.POINTER(_fp), C.POINTER(C.POINTER(C.c_uint32))]),
    "sph_world_read_surface_field": (C.c_int, [_vp, _fp, C.c_size_t, _fp, C.POINTER(C.c_uint32)]),
    "sph_surface_anisotropy_default": (None, [C.POINTER(SurfaceAnisotropy)]),
    "sph_world_extract_surface_anisotropic": (C.c_int, [_vp, C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(SurfaceDesc),
                                                        C.POINTER(SurfaceAnisotropy), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "sph_world_read_surface_ellipsoids": (C.c_int, [_vp, C.c_uint32, _fp, _fp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_map_surface_ellipsoids": (C.c_int, [_vp, C.c_uint32, C.POINTER(_fp), C.POINTER(_fp), C.POINTER(C.c_size_t)]),
    "sph_diffuse_desc_default": (None, [C.POINTER(DiffuseDesc)]),
    "sph_world_update_diffuse": (C.c_int, [_vp, C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(DiffuseDesc), C.c_float, _fp,
                                           C.POINTER(DiffuseStats)]),
    "sph_world_read_diffuse": (C.c_int, [_vp, _fp, _fp, _u8p, _fp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "sph_world_map_diffuse": (C.c_int, [_vp, C.POINTER(_fp), C.POINTER(_fp), C.POINTER(_u8p), C.POINTER(_fp), C.POINTER(C.c_size_t)]),
    "sph_world_clear_diffuse": (C.c_int, [_vp]),
}


def lib(kernels=False):
    """Load libsalva_b200.so (kernels=True: libsalva_b200_kernels.so, the build that carries the Poly6 / Spiky / Viscosity
    solver kernels); raises (never falls back) when it is missing."""
    global _LIB
    path = KERNELS_LIB_PATH if kernels else LIB_PATH
    if path not in _LIBS:
        if not os.path.exists(path):
            raise RuntimeError("%s is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); there is no CPU fallback"
                               % os.path.basename(path))
        L = C.CDLL(path)
        ab_build = bool(os.environ.get("SALVA_B200_LIB")) and not kernels  # A/B experiment builds may predate the newest entry points
        for name, (res, args) in SYMBOLS.items():
            if ab_build and not hasattr(L, name):
                continue
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _LIBS[path] = L
    if not kernels:
        _LIB = _LIBS[path]
    return _LIBS[path]
