"""Row order (SALVA_B200_XYSUB=2: x / y binned at h/2, one line of particles per bin column) against the default order and the oracle.

Row order runs its own grid kernels (k_cell_hist_xy, k_neighbors_xy, k_boundary_volumes_xy), and the benchmark picks it for C3
when it is faster, so a regression here is a regression of the timed workload.  The check runs in a SUBPROCESS with a timeout,
so that a crash or a hang of those kernels is reported as this test's failure, with the subprocess's output, instead of taking
the CUDA context of the session with it.  It checks exact contact counts and AABB query results in both orders, trajectories
equal to rounding, and both within the oracle tolerances.  tests/test_gpu_ref64.py and tests/test_gpu_ref64_fullsize.py check
the row order's passes one by one against the float64 reference.
"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CODE = r'''
import os, sys
import numpy as np
sys.path.insert(0, %(root)r)
from oracle.oracle import OracleWorld
from salva_b200 import DFSPHSolver, LiquidWorld, scenes

def scene(two_fluids):
    r = 0.05
    rng = np.random.default_rng(17)
    nx, ny, nz = 14, 11, 12
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, r * 0.93), r, 3, amplitude=0.3)
    vel = rng.normal(0, 0.2, pts.shape).astype(np.float32)
    tank = scenes.open_tank((-r, -r, -r), (nx * 2 * r + r, 1.2, nz * 2 * r + r), r)
    forces = [scenes.xsph_viscosity(0.5, 0.2), scenes.akinci2013_surface_tension(1.0, 0.5)]
    fluids = [dict(positions=pts, velocities=vel, density0=1000.0, forces=list(forces))]
    if two_fluids:
        up = scenes.jitter(scenes.block_lattice(nx, 4, nz, r * 0.93, origin=(0.0, ny * 2 * r * 0.93, 0.0)), r, 4, amplitude=0.3)
        fluids.append(dict(positions=up, velocities=rng.normal(0, 0.2, up.shape).astype(np.float32), density0=800.0, forces=list(forces)))
    lid = scenes._face(1, 1.2, (0.0, 0.0, 0.0), (0.6, 0.0, 0.5), 2 * r)          # a second boundary object
    return dict(particle_radius=r, fluids=fluids, boundaries=[dict(positions=tank, want_forces=True), dict(positions=lid)])

worst = 0.0
for two in (False, True):
    sc = scene(two)
    worlds = []
    for order in ("1", "2"):
        os.environ["SALVA_B200_XYSUB"] = order                       # read when the world is created
        w = LiquidWorld(DFSPHSolver(), particle_radius=sc["particle_radius"], smoothing_factor=2.0)
        worlds.append((w,) + scenes.populate(w, sc))
    cpu = OracleWorld(sc["particle_radius"], 2.0, solver=0)
    fc, bc = scenes.populate(cpu, sc)
    for w in [x[0] for x in worlds] + [cpu]:
        w.force_iterations(2, 3)
    for step in range(3):
        for w in [x[0] for x in worlds] + [cpu]:
            w.step(0.004)
        if step == 0:                                                 # identical inputs: integer work must agree exactly
            for k in range(len(fc)):
                ref_f, ref_b = cpu.debug(fc[k], "num_fluid_contacts"), cpu.debug(fc[k], "num_boundary_contacts")
                for w, fh, bh in worlds:
                    assert np.array_equal(w.debug(fh[k], "num_fluid_contacts"), ref_f)
                    assert np.array_equal(w.debug(fh[k], "num_boundary_contacts"), ref_b)
            assert worlds[0][0].stats()["n_contacts"] == worlds[1][0].stats()["n_contacts"] == cpu.stats()["n_contacts"]
    h = float(worlds[0][0].h)
    for k in range(len(fc)):
        pc, vc = cpu.read_fluid(fc[k])
        pa, va = worlds[0][0].read_fluid(worlds[0][1][k])
        pb, vb = worlds[1][0].read_fluid(worlds[1][1][k])
        assert np.abs(pa - pc).max() <= 1e-3 * h and np.abs(pb - pc).max() <= 1e-3 * h      # SURVEY 8(c)
        assert np.abs(pa - pb).max() <= 3e-4 * h                                            # the two orders differ by rounding only
        assert np.abs(worlds[1][0].debug(worlds[1][1][k], "density") - cpu.debug(fc[k], "density")).max() <= 1e-5 * 1000.0
        worst = max(worst, float(np.abs(pb - pc).max() / h))
    va_, _ = worlds[0][0].read_boundary(worlds[0][2][0])
    vb_, _ = worlds[1][0].read_boundary(worlds[1][2][0])
    assert np.abs(va_ - vb_).max() <= 1e-5 * np.abs(va_).max()                              # boundary volumes (k_boundary_volumes_xy)
    lo, hi = (0.1, 0.05, 0.1), (0.62, 0.4, 0.33)                                            # AABB query through the binned grid
    qa = worlds[0][0].particles_intersecting_aabb(lo, hi)
    qb = worlds[1][0].particles_intersecting_aabb(lo, hi)
    assert all(np.array_equal(x, y) for x, y in zip(qa, qb)) and len(qa[0]) > 50
    for w, _, _ in worlds:
        w.close()
print("ROW_ORDER_OK worst dx/h vs oracle %%.3e" %% worst)
'''


def test_row_order_matches_default_order_and_oracle():
    try:
        r = subprocess.run([sys.executable, "-c", CODE % {"root": ROOT}], capture_output=True, text=True, timeout=240, cwd=ROOT)
    except subprocess.TimeoutExpired as e:
        pytest.fail("row order did not finish within 240 s: " + str(e.stderr or e.stdout or "")[-600:])
    assert r.returncode == 0 and "ROW_ORDER_OK" in r.stdout, "row order failed: " + (r.stderr or r.stdout)[-600:]
    print(r.stdout.strip())
