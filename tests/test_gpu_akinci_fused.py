"""Akinci2013SurfaceTension on a single uniform-mass DFSPH fluid rides with the divergence loop: its normals with the first
velocity update (k_vel_update_u<.., NORMALS>) and its fluid term with the evaluation after it (k_vel_divergence_xsph_u<2>),
which the fold adds to gravity.  When no evaluation follows the update, or there is no update at all, or the force has a
boundary term, the separate passes compute it instead.  The force does not depend on velocities, so every path must give
the same acceleration."""
import numpy as np
import pytest

from oracle.oracle import OracleWorld
from salva_b200 import DFSPHSolver, LiquidWorld, scenes

pytestmark = pytest.mark.gpu

R = 0.05
DT = 0.004


def _scene(adhesion=0.0):
    nx, ny, nz, compress = 16, 12, 14, 0.95          # 2688 particles, ~5 % compressed
    rng = np.random.default_rng(17)
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, R * compress), R, 19, amplitude=0.2)
    vel = rng.normal(0, 0.2, pts.shape).astype(np.float32)
    tank = scenes.open_tank((-R, -R, -R), (nx * 2 * R * compress + R, 1.5, nz * 2 * R * compress + R), R)
    return dict(particle_radius=R, fluids=[dict(positions=pts, velocities=vel, density0=1000.0,
                                                forces=[scenes.akinci2013_surface_tension(1.0, adhesion)])],
                boundaries=[dict(positions=tank)])


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_every_akinci_path_gives_the_same_acceleration():
    sc = _scene()
    runs = {}
    for name, iters, max_div in [("no-update", (0, 1), None), ("fused", (1, 1), None), ("fused-then-plain", (3, 1), None),
                                 ("update-last", None, 1)]:
        solver = DFSPHSolver()
        if max_div is not None:
            solver.max_divergence_iter = max_div   # the loop ends with the normals-carrying update: no evaluation follows it
        w = LiquidWorld(solver, particle_radius=R, smoothing_factor=2.0)
        (f,), _ = scenes.populate(w, sc)
        if iters is not None:
            w.force_iterations(*iters)
        w.step(DT)
        if max_div is not None:
            assert w.stats()["n_divergence_iter"] == 1 and w.stats()["n_divergence_eval"] == 1
        runs[name] = w.debug(f, "acceleration")
        w.close()
    ref = runs["no-update"]
    assert np.abs(ref - np.array([0, -9.81, 0], np.float32)).max() > 1.0   # the force is acting
    for a in runs.values():
        np.testing.assert_array_max_ulp(a, ref, maxulp=1)


@pytest.mark.parametrize("adhesion", [0.0, 0.5], ids=["fused", "adhesion-fallback"])
def test_akinci_trajectory_matches_oracle(adhesion):
    sc = _scene(adhesion)
    gpu = LiquidWorld(DFSPHSolver(), particle_radius=R, smoothing_factor=2.0)
    cpu = OracleWorld(R, 2.0)
    (fg,), _ = scenes.populate(gpu, sc)
    (fc,), _ = scenes.populate(cpu, sc)
    for w in (gpu, cpu):
        w.force_iterations(2, 3)
    for step in range(5):
        gpu.step(DT)
        cpu.step(DT)
        if step == 0:   # lists built from identical positions; later steps may flip a pair sitting at |x_ij| = h
            assert np.array_equal(gpu.debug(fg, "num_fluid_contacts"), cpu.debug(fc, "num_fluid_contacts"))
            assert np.array_equal(gpu.debug(fg, "num_boundary_contacts"), cpu.debug(fc, "num_boundary_contacts"))
    h = float(gpu.h)
    assert _rel(gpu.debug(fg, "density"), cpu.debug(fc, "density")) <= 1e-5
    pg, _ = gpu.read_fluid(fg)
    pc, _ = cpu.read_fluid(fc)
    assert np.abs(pg - pc).max() <= 1e-3 * h
