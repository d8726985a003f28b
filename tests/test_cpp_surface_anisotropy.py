"""examples/surface_aniso3.cpp: basic3 for 100 steps, its anisotropic surface written as an OBJ.  Builds everywhere; on a GPU
its counts, volume and ellipsoid centres must match the Python mirror's extraction of the same scene."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _basic3_aniso(steps):
    """examples/surface_aniso3.cpp's scene through the Python mirror."""
    sys.path.insert(0, ROOT)
    from salva_b200 import LiquidWorld, SurfaceAnisotropy, scenes
    from oracle import ref64_surface as S
    r, n = 0.05, 15
    w = LiquidWorld(particle_radius=r)
    pts = scenes.cube_fluid(n, n, n, r)
    pts = (pts + np.array([0.0, np.float32(0.2) + np.float32(n) * np.float32(r), 0.0], np.float32)).astype(np.float32)
    f = w.add_fluid(pts)
    w.push_force(f, *scenes.artificial_viscosity(1.0, 0.0))
    i, k = np.meshgrid(np.arange(-25, 26), np.arange(-25, 26), indexing="ij")
    w.add_boundary(np.stack([np.float32(0.1) * i.ravel().astype(np.float32), np.full(i.size, 0.2, np.float32),
                             np.float32(0.1) * k.ravel().astype(np.float32)], axis=1))
    for _ in range(steps):
        w.step(np.float32(1.0 / 200.0))
    v, t, _ = w.surface_mesh(iso=0.6, anisotropy=SurfaceAnisotropy())
    c, _ = w.surface_ellipsoids(f)
    return len(c), float(c.astype(np.float64).sum()), len(v), len(t), S.volume(v, t)


def test_surface_aniso3_matches_the_python_mirror(tmp_path):
    import torch
    exe = str(tmp_path / "surface_aniso3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "surface_aniso3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    obj = str(tmp_path / "s.obj")
    run = subprocess.run([exe, "100", obj], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    words = run.stdout.replace(",", "").split()
    ne, nv, nt = (int(words[words.index(k) - 1]) for k in ("ellipsoids", "vertices", "triangles"))
    csum, vol = float(words[words.index("sum") + 1]), float(words[-1])
    pe, pcs, pv, pt, pvol = _basic3_aniso(100)
    assert (ne, nv, nt) == (pe, pv, pt)
    assert csum == pytest.approx(pcs, rel=1e-8)
    assert vol == pytest.approx(pvol, rel=1e-6)
    assert sum(1 for line in open(obj) if line.startswith("f ")) == nt
