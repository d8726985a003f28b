"""examples/heightfield3.cpp (heightfield3.rs): a heightfield ground surface-sampled on the device with the C++ mirror's
salva3d::sampling::shape_surface_ray_sample and coupled as a StaticSampling collider.  It builds everywhere and fails
loudly without a GPU.  On a GPU, after a few hundred steps:
- the ground boundary holds exactly the sampled points;
- nothing is NaN;
- no fluid particle over the footprint ends more than one particle radius below the triangulated surface;
- the Python mirror of the scene gives the same samples and the same fluid."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
F32 = np.float32
N = 41
STEPS = 300


def _build(tmp_path):
    exe = str(tmp_path / "heightfield3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "heightfield3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_heightfield_example_builds_and_fails_loudly_without_cuda(tmp_path):
    import torch
    exe = _build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    r = subprocess.run([exe, "1"], capture_output=True, text=True)
    assert r.returncode == 2 and "no CPU fallback" in r.stderr


def _python_mirror(heights):
    """heightfield3.rs:19-93 through the Python API."""
    from salva_b200 import BODY_FIXED, ArtificialViscosity, Fluid, LiquidWorld, StaticSampling, scenes
    from salva_b200 import sampling as S
    r = F32(0.15)
    w = LiquidWorld(particle_radius=0.15, smoothing_factor=2.0)
    try:
        pts = scenes.cube_fluid(15, 15, 15, r)
        pts[:, 1] += F32(1.0) + F32(15) * r * F32(2.0)
        fl = Fluid(pts, 0.15, 1000.0)
        fl.velocities = np.tile(np.array([0.0, -10.0, 0.0], F32), (len(pts), 1))
        fl.volumes = np.full(len(pts), r * r * r * F32(8.0 * 0.8), F32)  # fluid.rs:110-120
        fl.nonpressure_forces.append(ArtificialViscosity(1.0, 0.0))
        fh = w.add_fluid(fl)
        samples = S.shape_surface_ray_sample(w, S.HeightField(heights, (12.0, 1.0, 12.0)), r / F32(1.5))
        b = w.add_boundary(np.zeros((0, 3), F32))
        c = w.register_coupling(b, StaticSampling(samples))
        w.set_collider_state(c, body=BODY_FIXED)
        for _ in range(STEPS):
            w.step(1.0 / 200.0, (0.0, -9.81, 0.0))
        return samples, w.read_fluid(fh)[0]
    finally:
        w.close()


@pytest.mark.gpu
def test_heightfield_example_against_surface_and_python_mirror(tmp_path):
    from oracle import ref64_sampling as R
    exe = _build(tmp_path)
    dump = str(tmp_path / "hf3.bin")
    r = subprocess.run([exe, str(STEPS), dump], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    m = re.search(r"heightfield3: 3375 particles, (\d+) ground samples, boundary holds (\d+), %d steps, (\d+) non-finite" % STEPS, r.stdout)
    assert m, r.stdout
    n_samples, n_boundary, n_bad = (int(m.group(k)) for k in (1, 2, 3))
    assert n_samples > 5000 and n_boundary == n_samples and n_bad == 0, r.stdout

    raw = np.fromfile(dump, F32)
    heights = raw[:N * N].reshape(N, N)
    ns = int(raw[N * N])
    samples = raw[N * N + 1:N * N + 1 + 3 * ns].reshape(-1, 3)
    o = N * N + 1 + 3 * ns
    npart = int(raw[o])
    pos = raw[o + 1:o + 1 + 3 * npart].reshape(-1, 3)
    assert ns == n_samples and npart == 3375 and np.all(np.isfinite(pos))

    # heightfield3.rs:49-61 (simba's f32 sin / cos may differ from libm's in the last bit: compare to an f32 bound)
    i, j = np.meshgrid(np.arange(N), np.arange(N), indexing="ij")
    want = np.sin(i * 12.0 / 40) + np.cos(j * 12.0 / 40)
    want[[0, -1], :] = 3.0
    want[:, [0, -1]] = 3.0
    assert np.allclose(heights, want, atol=1e-6)

    # no particle over the footprint more than one radius below the triangulated surface
    hf = R._HF(R.Shape(R.HEIGHTFIELD, heights=heights, scale=(12.0, 1.0, 12.0)), ())
    inside = (np.abs(pos[:, 0]) <= 6.0) & (np.abs(pos[:, 2]) <= 6.0)
    below = [hf.height(float(p[0]), float(p[2])) - float(p[1]) for p in pos[inside]]
    assert inside.sum() > 0.5 * npart  # some of the splash leaves over the rim
    assert max(below) <= 0.15, max(below)

    py_samples, py_pos = _python_mirror(heights)
    assert np.array_equal(py_samples.view(np.uint32), samples.view(np.uint32))
    print("heightfield3: %d samples, deepest particle %.4f below the surface" % (ns, max(below)))
    assert np.array_equal(py_pos.view(np.uint32), pos.view(np.uint32))  # same library calls in the same order: bit-equal
