// basic3's scene (examples/basic3.cpp): its 15^3 block dropped onto its ground plane, with the whitewater of the splash as
// diffuse particles (DESIGN.md section 16).  Every frame (4 steps of 1/200 s) updates the diffuse set on the device and
// prints its counts; with an output prefix it also writes the set as "x y z vx vy vz kind life" lines, one file per frame.
//   g++ -std=c++17 -Iinclude examples/diffuse3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o diffuse3
//   ./diffuse3 [frames = 40] [out prefix, e.g. frames/diffuse]
#include <cstdio>
#include <cstdlib>
#include <string>

#include "salva3d_b200.hpp"

using namespace salva3d;

static Fluid cube_fluid(int ni, int nj, int nk, float particle_rad, float density) {
    std::vector<Point3> points;
    float hx = ni * particle_rad, hy = nj * particle_rad, hz = nk * particle_rad;
    for (int i = 0; i < ni; ++i)
        for (int j = 0; j < nj; ++j)
            for (int k = 0; k < nk; ++k)
                points.push_back({i * particle_rad * 2.0f + particle_rad - hx, j * particle_rad * 2.0f + particle_rad - hy,
                                  k * particle_rad * 2.0f + particle_rad - hz});
    return Fluid(points, particle_rad, density, InteractionGroups());
}

int main(int argc, char** argv) {
    const float PARTICLE_RADIUS = 0.05f, SMOOTHING_FACTOR = 2.0f, DT = 1.0f / 200.0f;
    const int frames = argc > 1 ? atoi(argv[1]) : 40, steps_per_frame = 4;
    const char* prefix = argc > 2 ? argv[2] : nullptr;
    try {
        LiquidWorld world(DFSPHSolver<>(), PARTICLE_RADIUS, SMOOTHING_FACTOR);
        const int n = 15;
        Fluid fluid = cube_fluid(n, n, n, PARTICLE_RADIUS, 1000.0f);
        for (auto& p : fluid.positions) p.y += 0.2f + n * PARTICLE_RADIUS;
        fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(1.0f, 0.0f));
        world.add_fluid(std::move(fluid));
        std::vector<Point3> ground;
        for (int i = -25; i <= 25; ++i)
            for (int k = -25; k <= 25; ++k) ground.push_back({i * 0.1f, 0.2f, k * 0.1f});
        world.add_boundary(Boundary(ground));
        const Vector3 g{0.0f, -9.81f, 0.0f};
        sph_diffuse_desc desc;
        sph_diffuse_desc_default(&desc);
        desc.lo[1] = 0.0f;  // particles that fall through the ground plane leave the set
        for (int frame = 0; frame < frames; ++frame) {
            for (int s = 0; s < steps_per_frame; ++s) world.step(DT, g);
            const sph_diffuse_stats st = world.update_diffuse(steps_per_frame * DT, g, &desc);
            printf("frame %d: emitted %llu dropped %llu expired %llu left %llu spray %llu foam %llu bubble %llu\n", frame,
                   (unsigned long long)st.emitted, (unsigned long long)st.dropped, (unsigned long long)st.expired, (unsigned long long)st.left_box,
                   (unsigned long long)st.spray, (unsigned long long)st.foam, (unsigned long long)st.bubble);
            if (!prefix) continue;
            const DiffuseParticles d = world.diffuse();
            const std::string path = std::string(prefix) + "_" + std::to_string(frame) + ".txt";
            FILE* f = fopen(path.c_str(), "w");
            if (!f) throw std::runtime_error("cannot write " + path);
            for (size_t i = 0; i < d.kinds.size(); ++i)
                fprintf(f, "%.7g %.7g %.7g %.7g %.7g %.7g %u %.7g\n", d.positions[i].x, d.positions[i].y, d.positions[i].z, d.velocities[i].x,
                        d.velocities[i].y, d.velocities[i].z, (unsigned)d.kinds[i], d.lives[i]);
            fclose(f);
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
