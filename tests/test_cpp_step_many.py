"""The C++ host mirror's LiquidWorld::step_many (include/salva3d_b200.hpp): builds everywhere; on a GPU, basic3 (C1) advanced
by one step_many(40) ends bit-identical to 40 calls of step."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"

SRC = r'''
#include <cstdio>
#include <cstring>
#include "salva3d_b200.hpp"
using namespace salva3d;
static LiquidWorld* basic3(FluidHandle* fh) {
    const float r = 0.05f;
    const int n = 15;
    auto* world = new LiquidWorld(DFSPHSolver<>(), r, 2.0f);
    std::vector<Point3> pts;
    const float hx = n * r;
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j)
            for (int k = 0; k < n; ++k) pts.push_back({i * r * 2.0f + r - hx, j * r * 2.0f + r - hx + 0.2f + n * r, k * r * 2.0f + r - hx});
    Fluid fluid(pts, r, 1000.0f, InteractionGroups());
    fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(1.0f, 0.0f));
    *fh = world->add_fluid(std::move(fluid));
    std::vector<Point3> ground;
    for (int i = -25; i <= 25; ++i)
        for (int k = -25; k <= 25; ++k) ground.push_back({i * 0.1f, 0.2f, k * 0.1f});
    world->add_boundary(Boundary(ground));
    return world;
}
int main() {
    try {
        const Vector3 g{0.0f, -9.81f, 0.0f};
        FluidHandle fa, fb;
        LiquidWorld* a = basic3(&fa);
        LiquidWorld* b = basic3(&fb);
        const uint32_t done = a->step_many(1.0f / 200.0f, g, 40);
        for (int s = 0; s < 40; ++s) b->step(1.0f / 200.0f, g);
        const Fluid& x = a->fluids()[fa];
        const Fluid& y = b->fluids()[fb];
        bool same = x.positions.size() == y.positions.size();
        for (size_t i = 0; same && i < x.positions.size(); ++i)
            same = !std::memcmp(&x.positions[i], &y.positions[i], sizeof(Point3)) && !std::memcmp(&x.velocities[i], &y.velocities[i], sizeof(Vector3));
        std::printf("done %u same %d\n", done, (int)same);
        delete a;
        delete b;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 2;
    }
    return 0;
}
'''


def test_cpp_step_many_builds_and_matches_step(tmp_path):
    import torch
    src = tmp_path / "step_many.cpp"
    src.write_text(SRC)
    exe = str(tmp_path / "step_many")
    r = subprocess.run([GXX, "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), str(src), "-L" + os.path.join(ROOT, "salva_b200"),
                        "-lsalva_b200", "-Wl,-rpath," + os.path.join(ROOT, "salva_b200"), "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device: built only")
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert r.stdout.split() == ["done", "40", "same", "1"], r.stdout
