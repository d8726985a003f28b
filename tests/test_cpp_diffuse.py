"""examples/diffuse3.cpp: basic3's block dropped onto its ground with diffuse particles per frame.  Builds everywhere; on a
GPU its per-frame counts must equal the Python mirror's for the same scene."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
FRAMES = 40


def _mirror(frames):
    """examples/diffuse3.cpp's scene and frames through the Python mirror: one stats dict per frame, and the last set."""
    sys.path.insert(0, ROOT)
    from salva_b200 import LiquidWorld, scenes
    r, n = 0.05, 15
    w = LiquidWorld(particle_radius=r)
    pts = scenes.cube_fluid(n, n, n, r)
    pts = (pts + np.array([0.0, np.float32(0.2) + np.float32(n) * np.float32(r), 0.0], np.float32)).astype(np.float32)
    f = w.add_fluid(pts)
    w.push_force(f, *scenes.artificial_viscosity(1.0, 0.0))
    i, k = np.meshgrid(np.arange(-25, 26), np.arange(-25, 26), indexing="ij")
    w.add_boundary(np.stack([np.float32(0.1) * i.ravel().astype(np.float32), np.full(i.size, 0.2, np.float32),
                             np.float32(0.1) * k.ravel().astype(np.float32)], axis=1))
    out = []
    dt = np.float32(1.0 / 200.0)
    for _ in range(frames):
        for _ in range(4):
            w.step(dt)
        out.append(w.update_diffuse(np.float32(4) * dt, (0.0, -9.81, 0.0), lo=(-np.inf, 0.0, -np.inf)))
    return out, w.diffuse_particles()


def test_diffuse3_matches_the_python_mirror(tmp_path):
    import torch
    exe = str(tmp_path / "diffuse3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "diffuse3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    prefix = str(tmp_path / "d")
    run = subprocess.run([exe, str(FRAMES), prefix], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    frames = [dict((k, int(v)) for k, v in re.findall(r"(\w+) (\d+)", line.split(":", 1)[1])) for line in run.stdout.splitlines()]
    stats, (p, v, kind, life) = _mirror(FRAMES)
    keys = {"emitted", "dropped", "expired", "left", "spray", "foam", "bubble"}
    want = [dict((("left" if k == "left_box" else k), s[k]) for k in s) for s in stats]
    assert [dict((k, fr[k]) for k in keys) for fr in frames] == want
    assert sum(s["emitted"] for s in stats) > 0, "the splash emitted nothing"
    last = np.loadtxt(prefix + "_%d.txt" % (FRAMES - 1), ndmin=2)
    assert len(last) == len(p)
    if len(p):
        assert np.array_equal(last[:, 6].astype(np.uint8), kind)
        assert np.allclose(last[:, :3], p, rtol=1e-6, atol=1e-6)
