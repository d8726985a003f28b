"""The C++ host mirror's substepping (LiquidWorld::set_substepping / substeps in include/salva3d_b200.hpp): builds
everywhere; on a GPU, (+inf, 3, 3) splits a step into three equal substeps."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"

SRC = r'''
#include <cmath>
#include <cstdio>
#include <limits>
#include "salva3d_b200.hpp"
using namespace salva3d;
int main() {
    try {
        LiquidWorld world(DFSPHSolver<>(), 0.05f, 2.0f);
        std::vector<Point3> pts;
        for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 6; ++j)
                for (int k = 0; k < 6; ++k) pts.push_back(Point3{0.1f * i, 0.1f * j, 0.1f * k});
        world.add_fluid(Fluid(pts, 0.05f, 1000.0f));
        world.set_substepping(std::numeric_limits<float>::infinity(), 3, 3);
        world.step(1.0f / 60.0f, Vector3{0.0f, -9.81f, 0.0f});
        std::vector<float> dts = world.substeps();
        std::printf("substeps %zu", dts.size());
        for (float dt : dts) std::printf(" %.9g", dt);
        std::printf("\n");
        world.set_substepping(0.4f, 0, 1);  // refused: min_substeps == 0
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
    return 0;
}
'''


def test_cpp_substepping_builds_and_runs(tmp_path):
    import torch
    src = tmp_path / "substeps.cpp"
    src.write_text(SRC)
    exe = str(tmp_path / "substeps")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), str(src), "-L" + os.path.join(ROOT, "salva_b200"),
                        "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2, (r.stdout, r.stderr)   # the refused setting throws
    words = r.stdout.split()
    assert words[:2] == ["substeps", "3"], r.stdout
    dts = [float(x) for x in words[2:]]
    assert all(abs(dt - 1.0 / 180.0) <= 1e-8 for dt in dts)
