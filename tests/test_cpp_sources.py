"""examples/faucet3_sources.cpp: faucet3's scene with a device source and sink, and with the same rule applied through the
host mirror's fluids_mut() (--host).  Builds everywhere; on a GPU both modes must print the same bookkeeping and checksum."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def test_faucet3_sources_matches_the_host_rule(tmp_path):
    import torch
    exe = str(tmp_path / "faucet3_sources")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "faucet3_sources.cpp"),
                        "-L" + os.path.join(ROOT, "salva_b200"), "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    dev = subprocess.run([exe, "300"], capture_output=True, text=True)
    host = subprocess.run([exe, "300", "--host"], capture_output=True, text=True)
    assert dev.returncode == 0 and host.returncode == 0, (dev.stderr, host.stderr)
    assert dev.stdout == host.stdout
    words = dev.stdout.split()
    assert int(words[words.index("removed") + 1].rstrip(",")) > 0  # the sheets reach the floor within 300 steps
