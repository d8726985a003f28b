"""Contact lists longer than the neighbour search's shared-memory staging (sph_kernels.cuh: NBR_SF = 32 fluid and NBR_SB = 8
boundary rows per particle): entries past those rows are stored straight to global memory, and the lists must still be exactly
the reference's, through a regrow of the list capacity and in a partial last warp."""
import numpy as np
import pytest

from oracle.oracle import OracleWorld
from salva_b200 import LiquidWorld, scenes

pytestmark = pytest.mark.gpu


def _exact_sets(pi, pj, h):
    """Per particle of pi, the sorted indices j of pj that pass the reference's test (dx*dx + dy*dy) + dz*dz <= h*h in f32."""
    h2 = np.float32(h) * np.float32(h)
    out = []
    for p in pi:
        d = p[None, :] - pj
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        out.append(np.flatnonzero(d2 <= h2).astype(np.uint32))
    return out


def test_lists_longer_than_the_staging_rows_match_the_reference():
    r = 0.05
    nx, ny, nz, compress = 13, 9, 11, 0.75          # 1287 particles (not a multiple of 32), ~2.4x rest density
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, r * compress), r, 23, amplitude=0.2)
    tank = scenes.open_tank((-r, -r, -r), (nx * 2 * r * compress + r, 1.0, nz * 2 * r * compress + r), r)
    sc = dict(particle_radius=r, fluids=[dict(positions=pts, velocities=np.zeros_like(pts), density0=1000.0, forces=[])],
              boundaries=[dict(positions=tank)])
    assert len(pts) % 32 != 0
    seen = {}

    def solve(ctx):
        ff, fb = ctx.fluid_fluid_contacts, ctx.fluid_boundaries_contacts
        seen["pos"] = ctx.positions.copy()
        seen["bpos"] = ctx.boundaries[0]["positions"].copy()
        seen["ff"] = [np.sort(ff.j[ff.offsets[i]:ff.offsets[i + 1]]) for i in range(len(ctx.positions))]
        seen["fb"] = [np.sort(fb.j[fb.offsets[i]:fb.offsets[i + 1]]) for i in range(len(ctx.positions))]
        seen["ff_models"] = np.unique(ff.j_model)
        seen["fb_models"] = np.unique(fb.j_model)

    gpu = LiquidWorld(particle_radius=r, smoothing_factor=2.0)
    (fg,), _ = scenes.populate(gpu, sc)
    gpu.push_host_force2(fg, solve)
    cpu = OracleWorld(r, 2.0)
    (fc,), _ = scenes.populate(cpu, sc)
    for w in (gpu, cpu):
        w.force_iterations(1, 1)
        w.step(1e-5)

    nf = gpu.debug(fg, "num_fluid_contacts").astype(np.int64)
    nb = gpu.debug(fg, "num_boundary_contacts").astype(np.int64)
    assert np.array_equal(nf, cpu.debug(fc, "num_fluid_contacts").astype(np.int64))     # exact, self included
    assert np.array_equal(nb, cpu.debug(fc, "num_boundary_contacts").astype(np.int64))
    # the scene reaches the paths it is written for
    assert gpu.stats()["max_neighbors"] > 64                  # beyond the initial capacity: the lists were regrown
    assert (nf > 32).mean() >= 0.25 and (nb > 8).sum() >= 32

    h = float(gpu.h)
    assert list(seen["ff_models"]) == [0] and list(seen["fb_models"]) == [0]
    want_f = _exact_sets(seen["pos"], seen["pos"], h)
    want_b = _exact_sets(seen["pos"], seen["bpos"], h)
    bad_f = [i for i in range(len(pts)) if not np.array_equal(seen["ff"][i], want_f[i])]
    bad_b = [i for i in range(len(pts)) if not np.array_equal(seen["fb"][i], want_b[i])]
    assert not bad_f, "fluid contact sets differ for %d particles, first %d" % (len(bad_f), bad_f[0])
    assert not bad_b, "boundary contact sets differ for %d particles, first %d" % (len(bad_b), bad_b[0])
