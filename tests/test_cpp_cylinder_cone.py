"""examples/cylinder_cone3.cpp: fluid poured onto a contact-sampled fixed cone and a cylinder on a dynamic body through the
C++ mirror.  It builds everywhere, fails loudly without a GPU, and on a GPU keeps the fluid out of both solids."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _build(tmp_path):
    exe = str(tmp_path / "cylinder_cone3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "cylinder_cone3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_cylinder_cone_example_builds_and_fails_loudly_without_cuda(tmp_path):
    import torch
    exe = _build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    r = subprocess.run([exe, "1"], capture_output=True, text=True)
    assert r.returncode == 2 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cylinder_cone_example_keeps_the_fluid_out(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe, "300"], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    m = re.search(r"cylinder_cone3: 800 particles, 300 steps, first samples at steps (-?\d+) and (-?\d+), (\d+) and (\d+) samples before, "
                  r"(\d+) and (\d+) empty steps after, (\d+) non-finite, deepest particle (\S+) inside, cylinder impulse \((\S+), (\S+), (\S+)\)",
                  r.stdout)
    assert m, r.stdout
    print("\n" + r.stdout.strip())
    f0, f1, b0, b1, e0, e1, nan = (int(m.group(k)) for k in range(1, 8))
    deepest = float(m.group(8))
    assert 0 < f0 < 300 and 0 < f1 < 300 and b0 == 0 and b1 == 0, r.stdout  # nothing before the fluid arrives, samples after
    assert nan == 0 and np.isfinite([float(m.group(k)) for k in (9, 10, 11)]).all()
    assert deepest <= 0.025, r.stdout  # no particle deeper inside either solid than one particle radius
