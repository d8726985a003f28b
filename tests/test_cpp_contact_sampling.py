"""examples/contact_sampling3.cpp: surface_tension3.rs with its ground coupled by DynamicContactSampling through the C++
mirror.  It builds everywhere, fails loudly without a GPU, and on a GPU the droplet rounds up on the sampled ground."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def _build(tmp_path):
    exe = str(tmp_path / "contact_sampling3")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "contact_sampling3.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_contact_sampling_example_builds_and_fails_loudly_without_cuda(tmp_path):
    import torch
    exe = _build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    r = subprocess.run([exe, "1"], capture_output=True, text=True)
    assert r.returncode == 2 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_contact_sampling_example_droplet_rests_on_the_sampled_ground(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe, "200"], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    m = re.search(r"contact_sampling3: 343 particles, 200 steps, radius of gyration ([0-9.e-]+) -> ([0-9.e-]+), lowest y = ([-0-9.e]+), "
                  r"ground samples (\d+)\.\.(\d+)", r.stdout)
    assert m, r.stdout
    g0, g1, lowest = (float(m.group(k)) for k in (1, 2, 3))
    smin, smax = int(m.group(4)), int(m.group(5))
    assert g1 < g0, r.stdout                      # surface tension rounds the cube up
    assert lowest >= 0.02 - 0.005, r.stdout        # no particle below the ground's top face minus r
    assert smin == 0 and smax > 0, r.stdout        # sampled only once the droplet comes near
