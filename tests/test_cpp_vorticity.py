"""examples/vorticity3.cpp: basic3 with vorticity confinement, printing the kinetic energy every 20 steps.  Builds everywhere;
on a GPU its output equals the Python mirror's, bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
F = np.float32


def _python_mirror(steps, eps):
    """examples/vorticity3.cpp's scene through the Python mirror: the lines it prints."""
    sys.path.insert(0, ROOT)
    from salva_b200 import LiquidWorld, scenes
    r, n = F(0.05), 15
    w = LiquidWorld(particle_radius=float(r))
    pts = scenes.cube_fluid(n, n, n, r)
    pts = (pts + np.array([0.0, F(0.2) + F(n) * r, 0.0], F)).astype(F)
    vol = F(F(r * r) * r) * F(8.0 * 0.8)   # Fluid::default_particle_volume
    mass = float(F(vol * F(1000.0)))
    f = w.add_fluid(pts, volumes=np.full(len(pts), vol, F))
    w.push_force(f, *scenes.artificial_viscosity(1.0, 0.0))
    w.push_force(f, *scenes.vorticity_confinement(eps))
    i, k = np.meshgrid(np.arange(-25, 26), np.arange(-25, 26), indexing="ij")
    w.add_boundary(np.stack([F(0.1) * i.ravel().astype(F), np.full(i.size, 0.2, F), F(0.1) * k.ravel().astype(F)], axis=1))
    lines = []
    for s in range(1, steps + 1):
        w.step(F(1.0 / 200.0))
        if s % 20 == 0:
            v = w.read_fluid(f)[1].astype(np.float64)
            e = 0.0
            for q in ((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]).tolist():
                e += mass * q
            lines.append("vorticity3: step %d kinetic energy %s" % (s, repr(0.5 * e)))
    return lines


def test_vorticity3_matches_the_python_mirror(tmp_path):
    import torch
    exe = str(tmp_path / "vorticity3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "vorticity3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    run = subprocess.run([exe, "100", "0.05"], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    got = [ln for ln in run.stdout.splitlines() if "kinetic energy" in ln]
    want = _python_mirror(100, 0.05)
    assert len(got) == 5
    # %.17g and repr both print the double's shortest round-trip digits or more: compare the values
    assert [float(g.split()[-1]) for g in got] == [float(x.split()[-1]) for x in want], (got, want)
