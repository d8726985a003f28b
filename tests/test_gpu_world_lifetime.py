"""A destroyed world gives back all the device memory it took, whatever features it used.

Each resource family runs in a subprocess of its own, so that it starts from a fresh CUDA context.  The subprocess runs one
warm-up cycle, because lazy module loading and first-use allocations take memory once, and then CYCLES cycles of create ->
exercise -> step -> destroy, reading the device's free memory after each.  Other processes share the GPU and move that figure
too, so the test bounds the median drop per cycle.  The host-force contacts, the mapped views and contact sampling are sized
so that a world that did not free their buffers would lose more than 16 MiB per cycle."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from salva_b200 import BODY_DYNAMIC, DynamicContactSampling, IISPHSolver, LiquidWorld, StaticSampling, scenes  # noqa: E402
from salva_b200 import sampling as S  # noqa: E402
from salva_b200.liquid_world import Ball, Cuboid  # noqa: E402

F32 = np.float32
R = 0.05
DT = 1.0 / 200.0
CYCLES = 8
MIB = float(1 << 20)
MAX_MEDIAN_DROP_MIB = 2.0


def _tank_world(n, solver=None, forces=()):
    """A jittered n x n x n block in an open tank."""
    w = LiquidWorld(solver=solver, particle_radius=R)
    pts = scenes.jitter(scenes.block_lattice(n, n, n, R), R, 7)
    side = 2 * R * n + R
    fh = w.add_fluid(pts)
    for kind, params in forces:
        w.push_force(fh, kind, params)
    w.add_boundary(scenes.open_tank((-R, -R, -R), (side, 2 * side, side), R))
    return w, fh


def _step(w, fh):
    w.step(DT)


def _elasticity(w, fh):
    w.step(DT)
    w.restore(w.snapshot())
    w.step(DT)


def _host_force(w, fh):
    seen = []
    w.push_host_force2(fh, lambda ctx: seen.append(int(ctx.fluid_fluid_contacts.j.shape[0])), contacts=True, boundaries=True)
    w.step(DT)
    assert seen and seen[-1] > 0


def _map(w, fh):
    w.map_positions(fh)
    w.step(DT)
    w.map_positions(fh)
    w.map_positions(fh, velocities=True)


def _static_collider(w, fh):
    c = w.register_coupling(w.add_boundary(np.zeros((0, 3), F32)), StaticSampling(scenes.cuboid_surface((0.2, 0.1, 0.2), R)))
    w.set_collider_state(c, translation=(0.5, 0.6, 0.5), body=BODY_DYNAMIC, linvel=(0.0, -1.0, 0.0), world_com=(0.5, 0.6, 0.5))
    w.step(DT)
    w.collider_impulse(c)


def _contact_world():
    """A 320 x 3 x 320 layer of fluid on a flat heightfield, every particle of it within the sampling distance, and a ball."""
    w = LiquidWorld(particle_radius=R)
    fh = w.add_fluid(scenes.block_lattice(320, 3, 320, R, origin=(-16.0, 0.0, -16.0)))
    hf = S.HeightField(np.zeros((8, 8), F32), (32.0, 1.0, 32.0))
    w.register_coupling(w.add_boundary(np.zeros((0, 3), F32)), DynamicContactSampling(hf))
    c = w.register_coupling(w.add_boundary(np.zeros((0, 3), F32)), DynamicContactSampling(Ball(0.3)))
    w.set_collider_state(c, translation=(0.0, 0.3, 0.0), body=BODY_DYNAMIC, linvel=(0.0, -1.0, 0.0), world_com=(0.0, 0.3, 0.0))
    return w, fh


def _contact(w, fh):
    w.step(DT)
    w.step(DT)


def _sample_shape(w, fh):
    S.shape_surface_ray_sample(w, Ball(0.3), R)
    S.shape_volume_ray_sample(w, Cuboid((0.2, 0.1, 0.3)), R)
    S.shape_surface_ray_sample(w, S.HeightField(np.linspace(0.0, 0.2, 36, dtype=F32).reshape(6, 6), (2.0, 1.0, 2.0)), R)
    w.step(DT)
    w.particles_intersecting_aabb((0.0, 0.0, 0.0), (0.5, 0.5, 0.5))
    w.particles_intersecting_shape(Ball(0.3), translation=(0.5, 0.5, 0.5))


# family -> (world builder, exercise); the builder returns (world, fluid handle)
FAMILIES = {
    "dfsph_tank": (lambda: _tank_world(20), _step),
    "iisph": (lambda: _tank_world(20, solver=IISPHSolver()), _step),
    "dfsph_viscosity": (lambda: _tank_world(20, forces=[scenes.dfsph_viscosity(0.5)]), _step),
    "becker2009": (lambda: _tank_world(16, forces=[scenes.becker2009_elasticity(1e5, 0.3)]), _elasticity),
    "he2014": (lambda: _tank_world(20, forces=[scenes.he2014_surface_tension(0.1)]), _step),
    "host_force_contacts": (lambda: _tank_world(32), _host_force),
    "map_views": (lambda: _tank_world(100), _map),
    "static_collider": (lambda: _tank_world(20), _static_collider),
    "contact_sampling": (_contact_world, _contact),
    "sample_shape": (lambda: _tank_world(20), _sample_shape),
}


def _child(family):
    import torch

    build, exercise = FAMILIES[family]
    free = []
    for _ in range(1 + CYCLES):
        w, fh = build()
        exercise(w, fh)
        w.close()
        free.append(torch.cuda.mem_get_info()[0])
    print("LIFETIME " + json.dumps({"family": family, "free": free}))


@pytest.mark.gpu
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_destroyed_world_returns_its_device_memory(family):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), family]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("LIFETIME ")][-1]
    free = json.loads(line[len("LIFETIME "):])["free"]
    drops = np.diff(np.asarray(free, np.float64)) * -1.0 / MIB  # the warm-up cycle is free[0]'s baseline, not a drop
    median = float(np.median(drops))
    print("%s: median drop %.2f MiB per cycle, drops %s" % (family, median, np.round(drops, 2).tolist()))
    assert median <= MAX_MEDIAN_DROP_MIB, "%s leaks %.2f MiB per cycle (drops %s MiB)" % (family, median, np.round(drops, 2).tolist())


if __name__ == "__main__":
    _child(sys.argv[1])
