"""Narrow (16-bit) fluid contact lists (sph_lists.cuh, DESIGN.md §4a.18): each entry is an offset into one of three stencil
windows, one per x-plane, of at most 2^14 slots.  A scene with a wider window repeats its search with 32-bit lists; the
width is chosen per search, so a world that leaves and re-enters the narrow range steps bit for bit as one that never left."""
import numpy as np
import pytest

from salva_b200 import LiquidWorld, scenes

pytestmark = pytest.mark.gpu

R = 0.05


@pytest.fixture(autouse=True)
def _h_cells(monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "1")  # narrow lists are written by the h-cell search


def _bits(w, f):
    b = np.unique(w.debug(f, "fluid_list_bits"))
    assert len(b) == 1
    return int(b[0])


def _column(n_layers, x0=0.0, mirror=False):
    """A column of 2 x 2 particles per layer at spacing 2r, n_layers layers along z: one z-column of h-cells (h = 4r).  The
    four sub-columns follow one another, the last one at x0 + 3r (mirror: at x0 + r)."""
    k = np.arange(n_layers, dtype=np.float32)
    pts = []
    for a in (0, 1):
        for b in (0, 1):
            p = np.zeros((n_layers, 3), np.float32)
            p[:, 0] = np.float32(x0) + np.float32((2 * (1 - a if mirror else a) + 1) * R)
            p[:, 1] = np.float32((2 * b + 1) * R)
            p[:, 2] = (k * np.float32(2.0) + np.float32(1.0)) * np.float32(R)
            pts.append(p)
    return np.concatenate(pts)


def _exact_sets_column(pos, h):
    """Per particle, the sorted indices j that pass the reference's test (dx*dx + dy*dy) + dz*dz <= h*h in f32, for a
    scene thin in x and y (one column, or a few side by side): candidates are those within h in z, found through the z
    order."""
    h2 = np.float32(h) * np.float32(h)
    order = np.argsort(pos[:, 2], kind="stable")
    zs = pos[order, 2]
    lo = np.searchsorted(zs, pos[:, 2] - np.float32(1.01 * h), side="left")
    hi = np.searchsorted(zs, pos[:, 2] + np.float32(1.01 * h), side="right")
    out = []
    for i in range(len(pos)):
        cand = order[lo[i]:hi[i]]
        d = pos[i][None, :] - pos[cand]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        out.append(np.sort(cand[d2 <= h2]).astype(np.uint32))
    return out


def test_a_window_wider_than_16_bits_takes_the_wide_lists_and_the_exact_sets():
    pts = scenes.jitter(_column(17000), R, 5, amplitude=0.2)  # 68 000 particles in one z-column of cells
    seen = {}

    def solve(ctx):
        ff = ctx.fluid_fluid_contacts
        seen["pos"] = ctx.positions.copy()
        seen["ff"] = [np.sort(ff.j[ff.offsets[i]:ff.offsets[i + 1]]) for i in range(len(ctx.positions))]

    w = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    f = w.add_fluid(pts, density0=1000.0)
    w.push_host_force2(f, solve, boundaries=False)
    w.force_iterations(1, 1)
    w.step(1e-5)
    assert _bits(w, f) == 32
    want = _exact_sets_column(seen["pos"], float(w.h))
    nf = w.debug(f, "num_fluid_contacts").astype(np.int64)
    assert np.array_equal(nf, [len(s) for s in want])
    bad = [i for i in range(len(pts)) if not np.array_equal(seen["ff"][i], want[i])]
    assert not bad, "fluid contact sets differ for %d particles, first %d" % (len(bad), bad[0])


def _three_columns(layers, extra=0):
    """Three columns (_column) in adjacent x-cells, jittered; `extra` more particles on top of the middle one.  The stencil
    window of every particle of the middle column in x-plane d is the whole of column d (the columns fill one y-row of
    cells), so its three windows span the three columns' sizes.  Returns the points and each point's column."""
    h = 4 * R
    cols = [_column(layers, 0.0), _column(layers, h), _column(layers, 2 * h, mirror=True)]
    if extra:
        top = np.float32((2 * layers + 1) * R)
        cols[1] = np.concatenate([cols[1], np.array([[h + R, R, top + k * 2 * R] for k in range(extra)], np.float32)])
    col = np.concatenate([np.full(len(c), k) for k, c in enumerate(cols)])
    return scenes.jitter(np.concatenate(cols), R, 13, amplitude=0.2), col


def _window_offsets(pts, col, sets):
    """Per plane d, the largest offset into column d (its window) of a contact of a middle-column particle, under the
    engine's sorted order: x-major cells, z fastest, and by particle id inside a cell (k_cell_sort)."""
    h = np.float32(4 * R)
    zc = np.floor((pts[:, 2] / h).astype(np.float32)).astype(np.int64)
    slot = np.empty(len(pts), np.int64)
    for k in range(3):
        idx = np.nonzero(col == k)[0]
        slot[idx[np.lexsort((idx, zc[idx]))]] = np.arange(len(idx))
    mid = np.nonzero(col == 1)[0]
    j = np.concatenate([sets[i] for i in mid]).astype(np.int64)
    return [int(slot[j[col[j] == d]].max()) for d in range(3)]


def _check_windows(pts, col, bits):
    """The exact contact sets through the host-force context, and density, alpha and the divergence sweep against the
    float64 reference on a row sample: the first and last layers of each column, the particles on top of the middle one,
    and 600 at random.  Returns the sets."""
    from oracle import ref64_stages as S
    seen = {}

    def solve(ctx):
        ff = ctx.fluid_fluid_contacts
        seen["pos"] = ctx.positions.copy()
        seen["ff"] = [np.sort(ff.j[ff.offsets[i]:ff.offsets[i + 1]]) for i in range(len(ctx.positions))]

    w = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    f = w.add_fluid(pts, density0=1000.0)
    w.push_host_force2(f, solve, boundaries=False)
    w.force_iterations(0, 0)
    w.step(1e-5)
    assert _bits(w, f) == bits
    w.close()
    assert np.array_equal(seen["pos"], pts)   # the context's rows are the caller's
    want = _exact_sets_column(pts, 4 * R)
    bad = [i for i in range(len(pts)) if not np.array_equal(seen["ff"][i], want[i])]
    assert not bad, "fluid contact sets differ for %d particles, first %d" % (len(bad), bad[0])

    rows = [np.random.default_rng(3).choice(len(pts), 600, replace=False)]
    for k in range(3):
        idx = np.nonzero(col == k)[0]
        z = pts[idx, 2]
        rows += [idx[np.argsort(z)[:8]], idx[np.argsort(z)[-8:]]]
    sc = dict(particle_radius=R, fluids=[dict(positions=pts, density0=1000.0,
                                             velocities=np.random.default_rng(5).normal(0, 0.2, pts.shape).astype(np.float32))],
              boundaries=[])
    c = S.Checks(lambda **kw: LiquidWorld(particle_radius=R, smoothing_factor=2.0), sc, rows=np.concatenate(rows))
    c.search()
    assert not c.flagged() and {"counts", "density", "alpha", "divergence_sweep"} <= set(c.worst), c.worst
    return want


def test_a_window_of_exactly_16384_slots_stays_narrow_and_reaches_every_offset():
    """Three columns of 16 384 particles (4 096 layers): the middle column's particles have three windows of exactly 2^14
    slots, the most a narrow list takes, and their contacts reach offset 0x3FFF in each (entries 0x3FFF, 0x7FFF, 0xBFFF)."""
    pts, col = _three_columns(4096)
    assert np.bincount(col).tolist() == [16384] * 3
    sets = _check_windows(pts, col, 16)
    assert _window_offsets(pts, col, sets) == [0x3FFF] * 3


def test_a_window_of_16385_slots_takes_the_wide_lists():
    pts, col = _three_columns(4096, extra=1)
    assert np.bincount(col).tolist() == [16384, 16385, 16384]
    sets = _check_windows(pts, col, 32)
    assert _window_offsets(pts, col, sets)[1] == 16384   # the slot past the narrow range is a contact


def test_a_window_of_40000_slots_takes_the_wide_lists():
    """Between 2^15 and 2^16 slots: the range a 15- or 16-bit offset would take, which the 68 000-slot column skips."""
    pts, col = _three_columns(10000)
    sets = _check_windows(pts, col, 32)
    assert min(_window_offsets(pts, col, sets)) >= 39990


def _block_scene():
    nx, ny, nz = 24, 16, 24
    pts = scenes.jitter(scenes.block_lattice(nx, ny, nz, R), R, 11)
    tank = scenes.open_tank((-R, -R, -R), (nx * 2 * R + R, 2.0, nz * 2 * R + R), R)
    return dict(particle_radius=R, fluids=[dict(positions=pts, density0=1000.0, forces=[scenes.xsph_viscosity(0.5, 0.0)])],
                boundaries=[dict(positions=tank)])


def test_a_lattice_block_stays_on_narrow_lists():
    w = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    (f,), _ = scenes.populate(w, _block_scene())
    w.step(1.0 / 200.0)
    assert _bits(w, f) == 16
    w.step_many(1.0 / 200.0, 3)
    assert _bits(w, f) == 16


def test_leaving_the_narrow_range_and_coming_back_steps_bit_for_bit():
    dt = 1.0 / 200.0
    a = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    b = LiquidWorld(particle_radius=R, smoothing_factor=2.0)
    (fa,), _ = scenes.populate(a, _block_scene())
    (fb,), _ = scenes.populate(b, _block_scene())
    for w in (a, b):  # pinned loops: the far column adds to the loop errors, not to any block particle's sums
        w.force_iterations(3, 3)
    for _ in range(2):
        a.step(dt)
    snap = a.snapshot()
    a.restore(snap)
    b.restore(snap)
    n = a.num_particles(fa)
    # b: a far column of the same fluid, wider than any narrow window, for two steps (one per-step, one in a step graph)
    col = scenes.jitter(_column(17000, x0=20.0), R, 7, amplitude=0.2)
    b.append_particles(fb, col)
    b.step(dt)
    assert _bits(b, fb) == 32
    b.step_many(dt, 2)
    assert _bits(b, fb) == 32
    mask = np.zeros(n + len(col), np.uint8)
    mask[n:] = 1
    b.delete_particles(fb, mask)
    b.step_many(dt, 3)
    assert _bits(b, fb) == 16
    # a: the same steps without the column
    a.step(dt)
    a.step_many(dt, 2)
    assert _bits(a, fa) == 16
    a.step_many(dt, 3)
    pa, va = a.read_fluid(fa)
    pb, vb = b.read_fluid(fb)
    assert np.array_equal(pa.view(np.uint32), pb.view(np.uint32))
    assert np.array_equal(va.view(np.uint32), vb.view(np.uint32))
