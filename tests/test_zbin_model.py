"""CPU model of the sub-divided cell bins of the neighbour search (salva_b200/csrc/sph_kernels.cuh: abin(), arun()).

Row order splits every cell of width h into `sub` slices along x and y and cuts each row of the 27-cell stencil down to the
slices within reach of the particle.  The claim that makes this safe — the contact sets stay EXACTLY the reference's
(contacts.rs:285: `(dx*dx + dy*dy) + dz*dz <= h*h` in f32, candidates from the 3 x 3 x 3 cells floor(x / h) +- 1) — is a
statement about f32 arithmetic, so it is checked here along one axis with numpy's IEEE f32 (same division, same floor,
directed rounding emulated through f64 + nextafter):

  * the bin is monotone in the coordinate and every bin lies inside ONE reference cell (bin // sub == floor(v / h));
  * whenever a pair passes the f32 distance test with the other two components zero (the worst case for this axis) and sits
    in adjacent reference cells, the partner's bin lies inside the run [lo, hi] the particle scans.
"""
import numpy as np
import pytest

F = np.float32


def abin(v, h, sub):
    q = F(v) / F(h)                      # __fdiv_rn
    fl = np.floor(q)
    s = int(F(q - fl) * F(sub))          # q - floor(q) is exact in f32; the product is rounded, hence the clamp
    return int(fl) * sub + min(sub - 1, s)


def _round_dir(x64, up):
    r = F(x64)
    if up and float(r) < x64:
        r = np.nextafter(r, F(np.inf))
    if not up and float(r) > x64:
        r = np.nextafter(r, F(-np.inf))
    return r


def arun(v, h, sub):
    c = int(np.floor(F(v) / F(h)))
    h_reach = np.nextafter(F(F(h) * F(1.00001)), F(np.inf))      # fill_static_consts(): Consts::h_reach
    vlo = _round_dir(float(F(v)) - float(h_reach), up=False)      # __fsub_rd
    vhi = _round_dir(float(F(v)) + float(h_reach), up=True)       # __fadd_ru
    lo = max(abin(vlo, h, sub), (c - 1) * sub)
    hi = min(abin(vhi, h, sub), (c + 2) * sub - 1)
    return lo, hi


def accepted(vi, vj, h):
    d = F(F(vi) - F(vj))
    return F(d * d) <= F(F(h) * F(h))                             # dist2_exact with the other two components zero


@pytest.mark.parametrize("sub", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("h", [0.1, 0.2, 0.37])
def test_zbin_is_monotone_and_nested_in_the_reference_cells(sub, h):
    rng = np.random.default_rng(sub * 7 + int(h * 100))
    v = np.sort(np.concatenate([rng.uniform(-40 * h, 40 * h, 4000), (np.arange(-60, 60) * h).astype(np.float64),
                                np.nextafter((np.arange(-60, 60) * F(h)).astype(F), F(-np.inf)).astype(np.float64)]).astype(F))
    bins = np.array([abin(x, h, sub) for x in v])
    assert np.all(np.diff(bins) >= 0)
    cells = np.floor(v / F(h)).astype(np.int64)
    assert np.array_equal(np.floor_divide(bins, sub), cells)


@pytest.mark.parametrize("sub", [2, 3, 4, 8])
@pytest.mark.parametrize("h", [0.1, 0.2, 0.37])
def test_no_accepted_pair_of_adjacent_cells_is_cut_off(sub, h):
    rng = np.random.default_rng(sub * 13 + int(h * 1000))
    checked = near = 0
    for scale in (1.0, 30.0, 3000.0):                              # far from the origin the f32 grid gets coarse
        vi_all = rng.uniform(-40 * h * scale, 40 * h * scale, 1500).astype(F)
        for vi in vi_all:
            # partners right at the cutoff (a few ulps either side) and anywhere within reach
            cands = [F(vi + s * F(h)) for s in (-1.0, 1.0)]
            for c in list(cands):
                x = c
                for _ in range(4):
                    x = np.nextafter(x, F(np.inf))
                    cands.append(x)
                x = c
                for _ in range(4):
                    x = np.nextafter(x, F(-np.inf))
                    cands.append(x)
            cands += list((vi + rng.uniform(-1.0, 1.0, 6) * h).astype(F))
            lo, hi = arun(vi, h, sub)
            ci = int(np.floor(F(vi) / F(h)))
            assert lo <= abin(vi, h, sub) <= hi
            for vj in cands:
                if not accepted(vi, vj, h):
                    continue
                cj = int(np.floor(F(vj) / F(h)))
                if abs(cj - ci) > 1:
                    continue                                       # the reference's stencil does not look there either
                checked += 1
                near += abs(abs(float(vi) - float(vj)) - h) < 1e-5 * h
                assert lo <= abin(vj, h, sub) <= hi, (vi, vj, lo, hi, abin(vj, h, sub))
    assert checked > 10000 and near > 1000
