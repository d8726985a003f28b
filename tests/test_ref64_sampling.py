"""CPU checks of the float64 ray-sampling reference (oracle/ref64_sampling.py): its closed-form cases, and that it flags
plausible sampler bugs, each applied to the reference itself."""
import numpy as np
import pytest

from oracle import ref64_sampling as R


def heightfield3_ground():
    """heightfield3.rs:46-61: 41 x 41, 3.0 on the rim, sin(i * 12 / 40) + cos(j * 12 / 40) inside, scale (12, 1, 12)."""
    n = 41
    H = np.zeros((n, n), np.float32)
    for i in range(n):
        for j in range(n):
            x = np.float32(i) * np.float32(12.0) / np.float32(n - 1)
            z = np.float32(j) * np.float32(12.0) / np.float32(n - 1)
            H[i, j] = 3.0 if i in (0, n - 1) or j in (0, n - 1) else np.sin(x) + np.cos(z)
    return R.Shape(R.HEIGHTFIELD, heights=H, scale=(12.0, 1.0, 12.0))


def bumpy_field(nr=9, nc=13):
    rng = np.random.default_rng(7)
    return R.Shape(R.HEIGHTFIELD, heights=rng.uniform(-1.0, 1.5, (nr, nc)).astype(np.float32), scale=(3.0, 1.0, 2.0))


@pytest.mark.parametrize("n,r", [((3, 4, 5), 0.25), ((1, 1, 1), 0.125), ((2, 7, 1), 0.5), ((6, 6, 6), 0.0625)])
def test_grid_aligned_cuboid_closed_form(n, r):
    sh = R.Shape(R.CUBOID, [k * r for k in n])
    surface, volume = R.cuboid_counts(n)
    s, v = R.sample(sh, r, False), R.sample(sh, r, True)
    assert len(s.undecided) == 0 and not s.lines and len(v.undecided) == 0 and not v.lines
    assert len(s.keys) == surface and len(v.keys) == volume
    c = R.unkey(v.keys)  # the box [1, n] of keys plus one layer past each far face
    assert c.min(axis=0).tolist() == [1, 1, 1] and c.max(axis=0).tolist() == [k + 1 for k in n]


def test_ball_known_cases():
    # radius sub: the rays through the centre's neighbours cross at +-sqrt(r^2 - sub^2) = 0; a ball smaller than the
    # grid's half spacing off every ray is missed entirely
    small = R.sample(R.Shape(R.BALL, [0.04]), 0.1, False)
    assert len(small.keys) == 0 and not small.lines
    one = R.sample(R.Shape(R.BALL, [0.07]), 0.1, False)  # only the axis-parallel rays at +-0.03 hit it
    assert len(one.keys) > 0 and len(one.undecided) == 0
    big = R.sample(R.Shape(R.BALL, [1.0]), 0.1, False)
    pts = R.unquantize(big.keys, big.origin, big.sub).astype(np.float64)
    rad = np.linalg.norm(pts, axis=1)
    assert np.all(np.abs(rad - 1.0) <= np.sqrt(3) * 0.2)  # within one grid diagonal of the sphere
    assert len(big.undecided) + len(big.lines) < 0.05 * len(big.keys)


def test_capsule_zero_half_height_is_a_ball():
    for vol in (False, True):
        a = R.sample(R.Shape(R.CAPSULE, [0.0, 0.45]), 0.1, vol)
        b = R.sample(R.Shape(R.BALL, [0.45]), 0.1, vol)
        assert np.array_equal(a.keys, b.keys) and np.array_equal(a.undecided, b.undecided)


def plateau_field():
    """7 x 7 heights: 0 on the rim, a 5 x 5 plateau at 0.1875 = 1.5 sub for particle_rad 0.0625.  The AABB's y starts at 0,
    so origin.y = -sub / 2: the plateau lies on the plane of the second row of horizontal rays, and vertical rays hit it at
    exactly 2 cells above origin (an integral ceil)."""
    H = np.zeros((7, 7), np.float32)
    H[1:6, 1:6] = 0.1875
    return R.Shape(R.HEIGHTFIELD, heights=H, scale=(1.5, 1.0, 1.5))


def test_plateau_on_a_ray_plane():
    s = R.sample(plateau_field(), 0.0625, False)
    c = R.unkey(s.keys)
    over = (c[:, 0] >= 3) & (c[:, 0] <= 10) & (c[:, 2] >= 3) & (c[:, 2] <= 10)  # vertical rays over the plateau, |x|, |z| < 0.5
    assert over.sum() > 0 and np.all(c[over & (c[:, 1] <= 2), 1] == 2)
    assert s.lines  # the horizontal rays in the plateau's plane are coplanar with its triangles: undecided from there on


def test_flat_heightfield_halfway_between_key_planes():
    sh = R.Shape(R.HEIGHTFIELD, heights=np.zeros((5, 5), np.float32), scale=(2.0, 1.0, 2.0))
    s = R.sample(sh, 0.125, False)
    c = R.unkey(s.keys)
    assert len(s.undecided) == 0 and not s.lines
    # the loosened AABB puts a flat field half a cell above origin, between two ray planes: only the vertical rays hit,
    # and ceil(0.5) = 1
    assert np.all(c[:, 1] == 1)
    assert len(s.keys) == 8 * 8  # the vertical rays over the closed footprint [-1, 1]^2 at spacing 0.25, off the rim
    assert len(R.sample(sh, 0.125, True).keys) == 0  # a surface has no volume: unpaired hits insert nothing


def test_heightfield3_ground_undecided_fraction_is_small():
    s = R.sample(heightfield3_ground(), 0.15 / 1.5, False)
    assert len(s.keys) > 5000
    assert len(s.undecided) + len(s.lines) < 0.02 * len(s.keys)


CASES = {
    "ceil_floor_swapped": (R.Shape(R.BALL, [1.0]), 0.1, False),
    "floor_across": (R.Shape(R.BALL, [1.0]), 0.1, False),
    "no_loosen": (R.Shape(R.CUBOID, [0.75, 0.5, 1.0]), 0.125, False),
    "no_half_offset": (R.Shape(R.CUBOID, [0.75, 0.5, 1.0]), 0.125, True),
    "times_sub": (R.Shape(R.CAPSULE, [20.0, 0.35]), 0.1, False),
    "no_skip": (R.Shape(R.CUBOID, [0.5, 0.005, 0.5]), 0.1, False),
    "skip_keeps_parity": (heightfield3_ground(), 0.1, False),  # horizontal rays grazing a crest cross twice within sub / 10
    "exclusive_end": (R.Shape(R.CUBOID, [0.75, 0.5, 1.0]), 0.125, True),
    "hf_zigzag": (bumpy_field(), 0.05, False),
    "hf_rows_along_x": (bumpy_field(), 0.05, False),
}


@pytest.mark.parametrize("bug", [b for b in R.BUGS if b != "fma_unquantize"])
def test_reference_flags_sampler_bug(bug):
    sh, r, vol = CASES[bug]
    good = R.sample(sh, r, vol)
    bad = R.sample(sh, r, vol, bugs=[bug])
    if bug == "times_sub":  # the rays themselves move: the capsule's 206th y-ray exists only with n * sub
        assert [len(t) for t in R.grid(sh, r)[3]] != [len(t) for t in R.grid(sh, r, [bug])[3]]
        assert bad.rays != good.rays
        return
    if bug in ("no_loosen", "no_half_offset"):  # a different grid: compare the points
        pg = R.unquantize(good.keys, good.origin, good.sub)
        pb = R.unquantize(bad.keys, bad.origin, bad.sub)
        assert len(pg) != len(pb) or not np.array_equal(pg, pb), bug
        return
    missing, unexplained, _ = R.compare(bad.keys, good)
    assert missing + unexplained > 0, bug


def test_reference_flags_fused_unquantize():
    s = R.sample(R.Shape(R.BALL, [1.3]), 0.1, True)
    good = R.unquantize(s.keys, s.origin, s.sub)
    bad = R.unquantize(s.keys, s.origin, s.sub, bugs=["fma_unquantize"])
    assert not np.array_equal(good.view(np.uint32), bad.view(np.uint32))


def test_keys_of_points_inverts_unquantize():
    s = R.sample(heightfield3_ground(), 0.1, False)
    assert np.array_equal(R.keys_of_points(R.unquantize(s.keys, s.origin, s.sub), s.origin, s.sub), s.keys)
