"""examples/surface3.cpp: basic3 for 100 steps, its surface written as an OBJ.  Builds everywhere; on a GPU its counts and
volume must match the Python mirror's mesh of the same scene."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _basic3_surface(steps):
    """examples/surface3.cpp's scene through the Python mirror."""
    sys.path.insert(0, ROOT)
    from salva_b200 import LiquidWorld, scenes
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
    v, t, _ = w.surface_mesh(iso=0.6)
    return len(v), len(t), S.volume(v, t)


def test_surface3_matches_the_python_mirror(tmp_path):
    import torch
    exe = str(tmp_path / "surface3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "surface3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    obj = str(tmp_path / "s.obj")
    run = subprocess.run([exe, "100", obj], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    words = run.stdout.replace(",", "").split()
    nv, nt, vol = int(words[words.index("vertices") - 1]), int(words[words.index("triangles") - 1]), float(words[-1])
    pv, pt, pvol = _basic3_surface(100)
    assert (nv, nt) == (pv, pt)
    assert vol == pytest.approx(pvol, rel=1e-6)
    assert sum(1 for line in open(obj) if line.startswith("f ")) == nt
