"""sph_world_sample_shape on the GPU against the float64 ray-sampling reference (oracle/ref64_sampling.py): the key set
outside the reference's undecided keys, bit-equal unquantised points, sorted and repeatable output, the cap / *n
contract, refusals that write nothing, and the closed-form count of a 10M-point cuboid."""
import ctypes as C

import numpy as np
import pytest

from oracle import ref64_sampling as R
from salva_b200 import LiquidWorld, SphError, _lib
from salva_b200 import sampling as S
from salva_b200.liquid_world import DFSPHSolver, Poly6Kernel

from test_ref64_sampling import bumpy_field, heightfield3_ground, plateau_field

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["lean", "kernels"])
def world(request):
    w = LiquidWorld(solver=DFSPHSolver(Poly6Kernel) if request.param == "kernels" else None, particle_radius=0.05)
    yield w
    w.close()


def _gpu_shape(sh):
    if sh.kind == R.HEIGHTFIELD:
        return S.HeightField(sh.heights, sh.scale)
    return {R.BALL: S.Ball, R.CUBOID: S.Cuboid, R.CAPSULE: S.Capsule}[sh.kind](*([list(sh.params)] if sh.kind == R.CUBOID else sh.params))


SHAPES = {
    "ball": R.Shape(R.BALL, [0.63]),
    "ball_below_sub": R.Shape(R.BALL, [0.07]),
    "cuboid": R.Shape(R.CUBOID, [0.4, 0.27, 0.55]),
    "cuboid_one_cell": R.Shape(R.CUBOID, [0.5, 0.05, 0.3]),
    "capsule": R.Shape(R.CAPSULE, [0.35, 0.22]),
    "capsule_zero_height": R.Shape(R.CAPSULE, [0.0, 0.31]),
    "heightfield_bumpy": bumpy_field(),
    "heightfield_2x2": R.Shape(R.HEIGHTFIELD, heights=np.array([[0.0, 0.4], [-0.3, 0.2]], np.float32), scale=(1.0, 1.0, 0.8)),
    "heightfield_flat": R.Shape(R.HEIGHTFIELD, heights=np.zeros((5, 7), np.float32), scale=(2.0, 1.0, 1.5)),
}
RADII = (0.05, 0.0625, 0.037)

_undecided = {}


def _check(world, sh, rad, volume):
    ref = R.sample(sh, rad, volume)
    fn = S.shape_volume_ray_sample if volume else S.shape_surface_ray_sample
    pts = fn(world, _gpu_shape(sh), rad)
    assert pts.dtype == np.float32 and pts.shape[1] == 3
    keys = R.keys_of_points(pts, ref.origin, ref.sub)
    # every coordinate is bit-equal to the unquantised key
    assert np.array_equal(pts.view(np.uint32), R.unquantize(keys, ref.origin, ref.sub).view(np.uint32))
    assert np.all(np.diff(keys) > 0)  # ascending keys, no duplicates
    missing, unexplained, und = R.compare(keys, ref)
    assert missing == 0 and unexplained == 0, (missing, unexplained, len(ref.keys))
    again = fn(world, _gpu_shape(sh), rad)
    assert np.array_equal(again.view(np.uint32), pts.view(np.uint32))
    return len(keys), und, len(ref.lines)


@pytest.mark.parametrize("volume", [False, True], ids=["surface", "volume"])
@pytest.mark.parametrize("rad", RADII)
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_matches_reference(world, name, rad, volume):
    n, und, lines = _check(world, SHAPES[name], rad, volume)
    _undecided[(name, volume)] = max(_undecided.get((name, volume), 0.0), (und + lines) / max(n, 1))
    print("%s %s r=%g: %d points, %d undecided keys, %d undecided ray tails" % (name, "volume" if volume else "surface", rad, n, und, lines))


def test_heightfield3_ground(world):
    n, und, lines = _check(world, heightfield3_ground(), 0.15 / 1.5, False)
    assert n > 5000
    print("heightfield3 ground: %d points, %d undecided keys, %d undecided ray tails" % (n, und, lines))


def test_plateau_on_a_ray_plane(world):
    """A plateau on the plane of a row of horizontal rays (coplanar with its triangles) and at an integral ceil for the
    vertical rays that hit it."""
    n, und, lines = _check(world, plateau_field(), 0.0625, False)
    pts = S.shape_surface_ray_sample(world, _gpu_shape(plateau_field()), 0.0625)
    top = pts[(np.abs(pts[:, 0]) < 0.5) & (np.abs(pts[:, 2]) < 0.5) & (pts[:, 1] > 0.1)]
    assert len(top) > 0 and np.all(top[:, 1] == np.float32(-0.0625) + np.float32(2) * np.float32(0.125))
    print("plateau: %d points, %d undecided keys, %d undecided ray tails" % (n, und, lines))


def _raw(world, method, shape, hf, rad, out, cap):
    n = C.c_size_t(12345)
    st = world._L.sph_world_sample_shape(world._w, method, C.byref(shape), C.byref(hf) if hf is not None else None, rad,
                                         out.ctypes.data_as(C.POINTER(C.c_float)) if out is not None else None, cap, C.byref(n))
    return st, n.value


def _cshape(kind, *p):
    s = _lib.Shape()
    s.kind = kind
    for a, v in enumerate(p):
        s.p[a] = v
    return s


def test_cap_and_count(world):
    full = S.shape_surface_ray_sample(world, S.Ball(0.3), 0.05)
    for cap in (0, 1, len(full) - 1, len(full), len(full) + 5):
        out = np.full((len(full) + 5, 3), -7.0, np.float32)
        st, n = _raw(world, 0, _cshape(1, 0.3), None, 0.05, out if cap else None, cap)
        assert st == 0 and n == len(full)
        k = min(cap, len(full))
        assert np.array_equal(out[:k], full[:k]) and np.all(out[k:] == -7.0)


def test_refusals_write_nothing(world):
    H = np.zeros((3, 3), np.float32)

    def hf(nr, nc, h=H, scale=(1.0, 1.0, 1.0)):
        f = _lib.HeightFieldC()
        f.nrows, f.ncols = nr, nc
        f.heights = h.ctypes.data_as(C.POINTER(C.c_float))
        f.scale[:] = scale
        return f

    bad_h = H.copy()
    bad_h[1, 1] = np.nan
    cases = [(_cshape(1, 0.3), None, 0.0), (_cshape(1, 0.3), None, -0.1), (_cshape(1, 0.3), None, float("nan")),
             (_cshape(1, 0.3), None, float("inf")), (_cshape(1, -0.3), None, 0.05), (_cshape(1, float("nan")), None, 0.05),
             (_cshape(2, 0.3, -1.0, 0.2), None, 0.05), (_cshape(3, 0.2, float("nan")), None, 0.05), (_cshape(7, 1.0), None, 0.05),
             (_cshape(4), hf(1, 3), 0.05), (_cshape(4), hf(3, 1), 0.05), (_cshape(4), hf(3, 3, bad_h), 0.05),
             (_cshape(4), hf(3, 3, scale=(1.0, 0.0, 1.0)), 0.05), (_cshape(4), hf(3, 3, scale=(-1.0, 1.0, 1.0)), 0.05),
             (_cshape(4), None, 0.05),
             (_cshape(2, 1.0e6, 1.0, 1.0), None, 0.1)]  # 2^21 or more cells along x
    for shape, f, rad in cases:
        for method in (0, 1):
            out = np.full((64, 3), 3.25, np.float32)
            st, n = _raw(world, method, shape, f, rad, out, 64)
            assert st == 1, (shape.kind, list(shape.p), rad)
            assert n == 12345 and np.all(out == 3.25)
    out = np.full((4, 3), 3.25, np.float32)
    st, _ = _raw(world, 2, _cshape(1, 0.3), None, 0.05, out, 4)
    assert st == 1 and np.all(out == 3.25)


def test_device_refuses_a_key_of_2_pow_21():
    """2^21 + 1 ray positions along x pass the host's check; the volume's last key along x is 2^21 and the device refuses
    it, while the surface's largest key is 2^21 - 1 and is sampled."""
    w = LiquidWorld(particle_radius=0.05)
    try:
        r = 2.0 ** -7
        nx = 2 ** 21 - 1
        shape = _cshape(2, nx * r, r, r)
        out = np.full((4, 3), 3.25, np.float32)
        st, n = _raw(w, 1, shape, None, r, out, 4)
        assert st == 1 and n == 12345 and np.all(out == 3.25)
        assert "2^21" in w._L.sph_last_error(w._w).decode()
        st, n = _raw(w, 0, shape, None, r, None, 0)
        assert st == 0 and n == R.cuboid_counts((nx, 1, 1))[0]
    finally:
        w.close()


def test_heightfield_kind_is_refused_elsewhere(world):
    n = C.c_size_t(0)
    t = (C.c_float * 3)(0, 0, 0)
    buf = (C.c_uint32 * 4)()
    st = world._L.sph_world_particles_in_shape(world._w, C.byref(_cshape(4)), t, None, buf, buf, buf, 4, C.byref(n))
    assert st == 1
    bh = world.add_boundary(np.zeros((1, 3), np.float32))
    c = C.c_uint32(0)
    assert world._L.sph_collider_register(world._w, bh, 1, C.byref(_cshape(4)), None, 0, C.byref(c)) == 1
    world.remove_boundary(bh)


def test_python_refusal_raises(world):
    with pytest.raises(SphError):
        S.shape_surface_ray_sample(world, S.Ball(0.3), 0.0)


def test_full_size_cuboid_closed_form():
    """A volume-sampled cuboid of 10M+ points: half extents n * r with a dyadic r make every operation exact."""
    w = LiquidWorld(particle_radius=0.05)
    try:
        n, r = (215, 216, 217), 2.0 ** -7
        surface, volume = R.cuboid_counts(n)
        pts = S.shape_volume_ray_sample(w, S.Cuboid([k * r for k in n]), r)
        assert len(pts) == volume and volume >= 10_000_000
        first = np.float32(-np.float32(n[0] * r) - np.float32(2 * r) + np.float32(r)) + np.float32(2 * r)  # key 1 along x
        assert pts[0, 0] == first
        surf = S.shape_surface_ray_sample(w, S.Cuboid([k * r for k in n]), r)
        assert len(surf) == surface
    finally:
        w.close()


def test_report_worst_undecided_fraction():
    for (name, vol), frac in sorted(_undecided.items()):
        print("worst undecided fraction %-22s %-7s %.4f" % (name, "volume" if vol else "surface", frac))
