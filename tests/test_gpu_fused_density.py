"""DFSPH's densities, alphas and first divergence evaluation are computed by the neighbour search itself, over the lists it has
just built (sph_kernels.cuh: density_alpha_div).  The first NBR_SF = 32 fluid and NBR_SB = 8 boundary entries of each list are
read from the search's shared-memory staging rows and the later ones back from global memory.  A compressed block makes the
lists longer than the staging rows and regrows the list capacity; 1287 particles leave a partial last warp."""
import numpy as np
import pytest

from oracle.oracle import OracleWorld
from salva_b200 import LiquidWorld, scenes
from salva_b200.liquid_world import SphError

pytestmark = pytest.mark.gpu

R = 0.05


def _compressed_scene(mass, density0=1000.0):
    nx, ny, nz, compress = 13, 9, 11, 0.75          # 1287 particles (not a multiple of 32), ~2.4x rest density
    rng = np.random.default_rng(7)
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, R * compress), R, 23, amplitude=0.2)
    vel = rng.normal(0, 0.2, pts.shape).astype(np.float32)
    if mass == "two_fluids":
        up = pts[:, 1] > np.median(pts[:, 1])
        fluids = [dict(positions=pts[~up], velocities=vel[~up], density0=density0),
                  dict(positions=pts[up], velocities=vel[up], density0=0.8 * density0)]
    else:
        vol = None
        if mass == "volumes":                       # per-particle masses: no uniform-mass records
            vol = ((2 * R) ** 3 * rng.uniform(0.8, 1.2, len(pts))).astype(np.float32)
        fluids = [dict(positions=pts, velocities=vel, density0=density0, volumes=vol)]
    tank = scenes.open_tank((-R, -R, -R), (nx * 2 * R * compress + R, 1.0, nz * 2 * R * compress + R), R)
    return fluids, tank


def _populate(world, fluids, tank):
    fh = [world.add_fluid(f["positions"], density0=f["density0"], velocities=f["velocities"], volumes=f.get("volumes"))
          for f in fluids]
    world.add_boundary(tank)
    return fh


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("order", ["h", "rows"])
@pytest.mark.parametrize("mass", ["uniform", "volumes", "two_fluids"])
def test_search_density_sweep_matches_oracle(mass, order, monkeypatch):
    if order == "rows":
        monkeypatch.setenv("SALVA_B200_XYSUB", "2")  # read when the world is created
    fluids, tank = _compressed_scene(mass)
    gpu = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    cpu = OracleWorld(R, 2.0)
    fg, fc = _populate(gpu, fluids, tank), _populate(cpu, fluids, tank)
    for w in (gpu, cpu):
        w.force_iterations(0, 0)                    # no velocity update: "divergence" is the evaluation the search computed
        w.step(1e-5)
    assert gpu.stats()["max_neighbors"] > 64        # beyond the initial capacity: the lists were regrown
    nf = np.concatenate([gpu.debug(f, "num_fluid_contacts") for f in fg]).astype(np.int64)
    nb = np.concatenate([gpu.debug(f, "num_boundary_contacts") for f in fg]).astype(np.int64)
    assert (nf > 32).mean() >= 0.25 and (nb > 8).sum() >= 32
    for f, o in zip(fg, fc):
        assert np.array_equal(gpu.debug(f, "num_fluid_contacts"), cpu.debug(o, "num_fluid_contacts"))
        assert np.array_equal(gpu.debug(f, "num_boundary_contacts"), cpu.debug(o, "num_boundary_contacts"))
        assert _rel(gpu.debug(f, "density"), cpu.debug(o, "density")) <= 1e-5
        assert _rel(gpu.debug(f, "alpha"), cpu.debug(o, "alpha")) <= 1e-5
        # the divergence cancels to ~1 % of its terms, so one ulp per term is amplified ~100x (DESIGN.md 4b)
        assert _rel(gpu.debug(f, "divergence"), cpu.debug(o, "divergence")) <= 1e-4


def test_zero_density_of_the_search_is_reported_as_zero_density():
    fluids, tank = _compressed_scene("uniform", density0=0.0)  # zero mass: every density is 0
    gpu = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    _populate(gpu, fluids, tank)
    gpu.force_iterations(0, 0)
    with pytest.raises(SphError, match="zero density") as e:
        gpu.step(1e-5)
    assert "boundary-volume" not in str(e.value)
