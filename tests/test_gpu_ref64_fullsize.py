"""The CUDA engine's passes against the float64 per-pass reference (oracle/ref64.py) at the paths only large scenes reach:
  - cell tables longer than 2048^2 entries, whose exclusive scan recurses to a third level (scan_exclusive): scattered
    scenes in a large box, one of them exactly 2048^2 + 1 entries long, every pass on every particle, in both orders;
  - C3 (10 077 696 particles, the benchmark's DFSPH + Akinci2013 workload, 7 % compressed, random velocities) in h order
    and in row order (whose table is longer than 2048^2): contact counts of every particle, every pass on a sample,
    boundary volumes of every boundary particle, and both loop errors over 78 732 pass blocks against the bound of the
    reduction tree the kernels run (ref64.structural_depth);
  - C5 (2 000 000 particles, IISPH, two fluids, artificial viscosity and Becker2009) on a sample spanning both fluids and
    the interface between them;
  - C2 (1 000 000 particles) in row order.
The sample (ref64_stages.full_size_rows): seeded random particles, every particle with a boundary contact, the particles of
the first and the last occupied cell, and those of the cells at the scan's block and level seams (table index within 2 of
a multiple of 2048 or 2048^2).  Each test prints the worst |err| / bound per pass and the excluded counts."""
import json
import time

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import ref64_stages as S
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, scenes

pytestmark = pytest.mark.gpu

F = np.float32
ORDERS = {"h_order": 1, "row_order": 2}
SCAN2 = S.SCAN_B * S.SCAN_B


def _make(r, solver=DFSPHSolver):
    def make(**kw):
        s = solver()
        for k, v in kw.items():
            setattr(s, k, v)
        return LiquidWorld(s, particle_radius=r, smoothing_factor=2.0)
    return make


def _report(c, **tags):
    print("\nREF64 %s" % json.dumps(dict(tags, worst={k: round(float(v), 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v})))
    assert not c.flagged(), c.flagged()


def _h(r):
    return F(F(r) * F(2.0) * F(2.0))


def _table_length(stats, xysub):
    return int(np.prod(stats["grid_dims"], dtype=np.int64)) * xysub * xysub + 1


# ---- cell tables past 2048^2 with few particles ------------------------------------------------------------------------------
def scene_corners(dims):
    """Two small jittered blocks (6 x 6 x 6 at 0.8 spacing, each on a floor plate) at opposite corners of a box whose grid
    is `dims` cells of width h: by the engine's rule dims = (max cell - min cell) + 3, the low block's cells start at 1
    and the high block's end at dims - 2."""
    r, h = S.R, float(_h(S.R))
    top = np.asarray(dims, np.float64) - 2
    fluids, plates = [], []
    for k, o in enumerate((np.array([0.3, 0.34, 0.3]), (top + 0.5) * h - 0.45)):
        pts = scenes.jitter(scenes.block_lattice(6, 6, 6, r * 0.8, origin=tuple(o)), r, 51 + k, amplitude=0.2)
        fluids.append(pts)
        plates.append(scenes._face(1, o[1] - 0.08, (o[0] - 0.02, 0.0, o[2] - 0.02), (o[0] + 0.48, 0.0, o[2] + 0.48), 2 * r))
    pts = np.concatenate(fluids).astype(F)
    plate = np.concatenate(plates).astype(F)
    return dict(fluids=[S._fluid(pts, 53)], boundaries=[dict(positions=plate, velocities=S._bvel(len(plate), 55))])


# (grid dims, table length): past 2048^2, and exactly 2048^2 + 1 (2049 level-0 blocks, the last holding one entry, and a
# level-1 scan of two blocks)
SCAN_SCENES = {
    ("h_order", "past"): ((150, 140, 260), None),
    ("h_order", "exact"): ((128, 128, 256), SCAN2 + 1),
    ("row_order", "past"): ((150, 140, 260), None),
    ("row_order", "exact"): ((64, 128, 128), SCAN2 + 1),
}


@pytest.mark.parametrize("order,kind", sorted(SCAN_SCENES), ids=["-".join(k) for k in sorted(SCAN_SCENES)])
def test_every_pass_on_a_cell_table_past_2048_squared(order, kind, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", str(ORDERS[order]))   # read when the world is created
    dims, length = SCAN_SCENES[(order, kind)]
    sc = scene_corners(dims)
    xs = ORDERS[order]
    _, mdims, mlen = S.cell_table(sc["fluids"][0]["positions"], sc["boundaries"][0]["positions"], _h(S.R), xs)
    assert list(mdims) == list(dims)
    c = S.Checks(_make(S.R), sc)
    o = c.stages()
    got = _table_length(o["stats"], xs)
    assert list(o["stats"]["grid_dims"]) == list(dims) and got == mlen
    assert got > SCAN2 and (length is None or got == length), got
    c.loop_errors()
    if kind == "exact":
        ci = S.Checks(_make(S.R, IISPHSolver), sc)
        ci.iisph_stages()
        _report(ci, scene="corners_" + kind, order=order, solver="iisph", table=got)
    _report(c, scene="corners_" + kind, order=order, table=got)
    assert c.worst["counts"] == 0


# ---- C3 at full size -------------------------------------------------------------------------------------------------------
def _full_scene(base, seed):
    """A bench scene with seeded random velocities (sigma 0.2 m/s) and still boundaries, forces left to the checks."""
    rng = np.random.default_rng(seed)
    fl = [dict(positions=f["positions"], velocities=rng.normal(0, 0.2, f["positions"].shape).astype(F), density0=f["density0"])
          for f in base["fluids"]]
    bd = [dict(positions=b["positions"], velocities=np.zeros_like(b["positions"])) for b in base["boundaries"]]
    return dict(particle_radius=base["particle_radius"], dt=base["dt"], fluids=fl, boundaries=bd)


def _counts_and_rows(sc, xysub, n_random, seed, extra=()):
    """Exact contact counts of every particle, the model of the cell table, and the sample."""
    P = np.concatenate([f["positions"] for f in sc["fluids"]]).astype(F)
    B = np.concatenate([b["positions"] for b in sc["boundaries"]]).astype(F)
    h = _h(sc["particle_radius"])
    nf, edge_f = S.exact_counts(P, P, h, tree=cKDTree(P.astype(np.float64)))
    nb, edge_b = S.exact_counts(P, B, h)
    idx, dims, length = S.cell_table(P, B, h, xysub)
    rows = S.full_size_rows(idx, nb, n_random, seed)
    if len(extra):
        rows = np.union1d(rows, extra)
    return P, nf, nb, dims, length, rows, dict(edge_pairs=edge_f + edge_b, sample=len(rows), tank=int((nb > 0).sum()),
                                               table=length)


@pytest.mark.parametrize("order", ["h_order", "row_order"])
def test_c3_full_size_every_pass_against_ref64(order, monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", str(ORDERS[order]))
    t0 = time.time()
    xs = ORDERS[order]
    sc = _full_scene(scenes.scene_c3(compress=0.93), 0xC3)
    n = len(sc["fluids"][0]["positions"])
    assert n == 10_077_696
    P, nf, nb, dims, length, rows, info = _counts_and_rows(sc, xs, 20_000, 3)
    make = _make(sc["particle_radius"])
    c = S.Checks(make, sc, rows=rows)
    o = c.stages()
    # contact counts of every particle, fluid and boundary
    assert np.array_equal(o["num_fluid_contacts"], nf) and np.array_equal(o["num_boundary_contacts"], nb)
    assert list(o["stats"]["grid_dims"]) == list(dims) and _table_length(o["stats"], xs) == length
    if xs > 1:
        assert length > SCAN2, length
    # boundary volumes of every boundary particle (Checks: the boundary contacts stay complete in rows mode)
    assert "boundary_volume" in c.worst
    # both loop errors over every particle, against the reduction tree's bound, with more than 65 536 pass blocks
    assert -(-n // S.PASS_T) > 65_536
    depth = c.loop_errors_read()
    assert {"divergence_error_read_1_blind_to_lost_blocks", "divergence_error_read_2_blind_to_lost_blocks"} <= set(c.worst)
    # Akinci2013 (1, 0), fused into the update and the evaluation after it, on a sub-sample: its normals need the
    # neighbours' lists too
    ak = S.Checks(make, sc, rows=np.random.default_rng(4).choice(rows, 4000, replace=False))
    ak.akinci(0.0)
    c.worst.update(ak.worst)
    c.excluded.update(ak.excluded)
    _report(c, scene="c3", order=order, n=n, depth=depth, akinci_sample=4000, seconds=round(time.time() - t0), **info)


# ---- C5 at full size -------------------------------------------------------------------------------------------------------
def test_c5_full_size_iisph_artificial_becker_against_ref64():
    t0 = time.time()
    base = scenes.scene_c5()
    sc = _full_scene(base, 0xC5)
    n0 = len(sc["fluids"][0]["positions"])
    P = np.concatenate([f["positions"] for f in sc["fluids"]])
    y_iface = float(base["fluids"][1]["positions"][:, 1].min() + base["fluids"][0]["positions"][:, 1].max()) / 2
    iface = np.nonzero(np.abs(P[:, 1] - y_iface) <= float(_h(sc["particle_radius"])))[0]
    _, nf, nb, dims, length, rows, info = _counts_and_rows(sc, 1, 20_000, 5, extra=iface)
    fid = np.r_[np.zeros(n0, int), np.ones(len(P) - n0, int)]
    assert len(P) == 2_000_000
    assert (fid[rows] == 0).sum() >= 10_000 and (fid[rows] == 1).sum() >= 10_000 and len(iface) >= 10_000
    c = S.Checks(_make(sc["particle_radius"], IISPHSolver), sc, rows=rows)
    o = c.iisph_stages()
    assert np.array_equal(o["num_fluid_contacts"], nf) and np.array_equal(o["num_boundary_contacts"], nb)
    c.artificial(1.0, 0.0, iisph=True)
    c.becker_capture(1.0e5, 0.3, True)
    assert {"dii", "aii", "dij_pjl", "pressure_1", "pressure_2", "velocity", "pressure_warm", "artificial_no_update",
            "el_volume", "el_capture_nonlinear_rotation", "el_capture_nonlinear_grad_tr", "el_capture_nonlinear_stress",
            "el_capture_nonlinear_force"} <= set(c.worst)
    _report(c, scene="c5", n=len(P), interface=len(iface), seconds=round(time.time() - t0), **info)


# ---- C2 at full size in row order ------------------------------------------------------------------------------------------
def test_c2_full_size_row_order_against_ref64(monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "2")
    t0 = time.time()
    sc = _full_scene(scenes.scene_c2(compress=0.93), 0xC2)
    _, nf, nb, dims, length, rows, info = _counts_and_rows(sc, 2, 20_000, 7)
    c = S.Checks(_make(sc["particle_radius"]), sc, rows=rows)
    o = c.stages()
    assert np.array_equal(o["num_fluid_contacts"], nf) and np.array_equal(o["num_boundary_contacts"], nb)
    assert list(o["stats"]["grid_dims"]) == list(dims) and _table_length(o["stats"], 2) == length
    _report(c, scene="c2", order="row_order", n=len(nf), seconds=round(time.time() - t0), **info)
