"""examples/colliders3.cpp: the C++ mirror's collider coupling (a StaticSampling tank on a fixed body and a ball on a dynamic
body the example integrates from the returned impulses) builds everywhere, fails loudly without a GPU, and on a GPU the
fluid stops the falling ball."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _build(tmp_path):
    exe = str(tmp_path / "colliders3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "colliders3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_colliders_example_builds_and_fails_loudly_without_cuda(tmp_path):
    import torch
    exe = _build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    r = subprocess.run([exe, "1"], capture_output=True, text=True)
    assert r.returncode == 2 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_colliders_example_couples_both_ways(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe, "80"], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    m = re.search(r"colliders3: 1728 particles, (\d+) tank samples, 80 steps, ball y = ([-0-9.e]+) \(lowest ([-0-9.e]+)\), vy = ([-0-9.e]+), "
                  r"max \|impulse\| = ([-0-9.e]+)", r.stdout)
    assert m, r.stdout
    y, lowest, vy, imp = (float(m.group(k)) for k in (2, 3, 4, 5))
    assert int(m.group(1)) > 0 and imp > 0.0
    # in free fall from y = 1.9 at 3 m/s down the ball would be at 1.9 - 3 * 0.4 - 9.81 * 0.4^2 / 2 = -0.085 after 80 steps:
    # the fluid's impulses hold it well above that, above the ground (y = 0.2 + radius)
    assert lowest > 0.45 and y > 0.45, r.stdout
