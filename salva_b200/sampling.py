"""salva3d::sampling (sampling/ray_sampling.rs:9-231) on the GPU: ray sampling of a shape's surface or volume into particle
positions, in the shape's local frame.

The reference signatures take (shape, particle_rad); these take the LiquidWorld first, whose device, stream and scratch
memory run the sampler (the world's particles are not touched).  Points come back as an (n, 3) float32 array in ascending
order of their quantised (x, y, z) keys, where the reference returns HashSet order.  DESIGN.md section 11.
"""
import ctypes as C

import numpy as np

from . import _lib
from .liquid_world import Ball, Capsule, Cone, Cuboid, Cylinder, heightfield_c  # noqa: F401  (the shapes the sampler takes, with HeightField)

SURFACE, VOLUME = 0, 1  # SPH_SAMPLE_*


class HeightField:
    """parry HeightField(heights, scale): rows of `heights` run along z and columns along x, the field spans
    [-0.5, 0.5] * scale in x and z, heights are multiplied by scale[1], and each cell is split along its (x0, z1)-(x1, z0)
    diagonal.  Also a collider shape for DynamicContactSampling and LiquidWorld.particles_intersecting_shape."""
    kind = 4

    def __init__(self, heights, scale):
        self.heights = np.ascontiguousarray(heights, np.float32)
        if self.heights.ndim != 2:
            raise ValueError("heights must be a 2-D (nrows, ncols) matrix")
        self.scale = [float(s) for s in scale]
        self.params = []


def _ray_sample(world, shape, particle_rad, method):
    sh = _lib.Shape()
    sh.kind = shape.kind
    for a, p in enumerate(shape.params):
        sh.p[a] = p
    hf = heightfield_c(shape) if shape.kind == HeightField.kind else None
    n = C.c_size_t(0)
    cap = getattr(world, "_sample_cap", 1 << 16)
    while True:
        out = np.empty((cap, 3), np.float32)
        world._ck(world._L.sph_world_sample_shape(world._w, method, C.byref(sh), C.byref(hf) if hf is not None else None,
                                                  particle_rad, out.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n)))
        if n.value <= cap:
            world._sample_cap = max(cap, n.value)
            return out[:n.value].copy()
        cap = n.value


def shape_surface_ray_sample(world, shape, particle_rad):
    """ray_sampling.rs:9-15: points on the surface of `shape` (Ball, Cuboid, Capsule, Cylinder, Cone or HeightField)."""
    return _ray_sample(world, shape, particle_rad, SURFACE)


def shape_volume_ray_sample(world, shape, particle_rad):
    """ray_sampling.rs:17-24: points filling the volume of `shape`."""
    return _ray_sample(world, shape, particle_rad, VOLUME)
