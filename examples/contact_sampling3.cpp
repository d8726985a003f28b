// examples3d/surface_tension3.rs (surface_tension3.rs:21-95) as written, on the C++ host mirror without the rapier testbed:
// a 1 cm^3 droplet (7^3 particles of radius 0.005, length unit 1 dm, gravity -0.981) with Akinci2013SurfaceTension(1, 0) +
// ArtificialViscosity(0.01, 0.01) falls onto a fixed cuboid ground (half extents 0.15, 0.02, 0.15) coupled by
// ColliderSampling::DynamicContactSampling: every step the library samples the ground where the droplet is about to touch
// it and pushes penetrating particles out.  Prints the droplet's radius of gyration before and after, its lowest particle
// height and the range of the ground's sample count over the run.
//   g++ -std=c++17 -Iinclude examples/contact_sampling3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o contact_sampling3
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "salva3d_b200.hpp"

using namespace salva3d;

static double gyration(const std::vector<Point3>& pts) {
    double cx = 0, cy = 0, cz = 0;
    for (auto& p : pts) { cx += p.x; cy += p.y; cz += p.z; }
    const double n = (double)pts.size();
    cx /= n; cy /= n; cz /= n;
    double s = 0;
    for (auto& p : pts) s += (p.x - cx) * (p.x - cx) + (p.y - cy) * (p.y - cy) + (p.z - cz) * (p.z - cz);
    return std::sqrt(s / n);
}

int main(int argc, char** argv) {
    const float PARTICLE_RADIUS = 0.005f, SMOOTHING_FACTOR = 2.0f;
    const int steps = argc > 1 ? std::atoi(argv[1]) : 200;
    try {
        LiquidWorld world(DFSPHSolver<>(), PARTICLE_RADIUS, SMOOTHING_FACTOR);
        std::vector<Point3> pts;  // helper::cube_fluid(7, 7, 7, r, 1000) translated by (0, 0.08, 0)
        const int n = 7;
        const float half = n * PARTICLE_RADIUS;
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j)
                for (int k = 0; k < n; ++k)
                    pts.push_back({i * PARTICLE_RADIUS * 2.0f + PARTICLE_RADIUS - half, j * PARTICLE_RADIUS * 2.0f + PARTICLE_RADIUS - half + 0.08f,
                                   k * PARTICLE_RADIUS * 2.0f + PARTICLE_RADIUS - half});
        const double g0 = gyration(pts);
        Fluid fluid(pts, PARTICLE_RADIUS, 1000.0f, InteractionGroups());
        fluid.nonpressure_forces.push_back(std::make_shared<Akinci2013SurfaceTension>(1.0f, 0.0f));
        fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(0.01f, 0.01f));
        const FluidHandle fh = world.add_fluid(std::move(fluid));
        // the ground: a cuboid collider on a fixed body at the origin, its boundary empty until the first step samples it
        const BoundaryHandle bh = world.add_boundary(Boundary({}));
        const ColliderHandle ground = world.register_coupling(bh, ColliderSampling::DynamicContactSampling(Cuboid{Vector3{0.15f, 0.02f, 0.15f}}));
        world.set_collider_state(ground, Isometry3(), SPH_BODY_FIXED);
        size_t smin = SIZE_MAX, smax = 0;
        for (int s = 0; s < steps; ++s) {
            world.step(1.0f / 200.0f, Vector3{0.0f, -0.981f, 0.0f});
            const size_t m = world.boundaries()[bh].num_particles();
            smin = std::min(smin, m);
            smax = std::max(smax, m);
        }
        const Fluid& f = world.fluids()[fh];
        float lowest = INFINITY;
        for (auto& p : f.positions) lowest = std::min(lowest, p.y);
        std::printf("contact_sampling3: %zu particles, %d steps, radius of gyration %.6f -> %.6f, lowest y = %.6f, ground samples %zu..%zu\n",
                    f.num_particles(), steps, g0, gyration(f.positions), lowest, steps ? smin : 0, smax);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "contact_sampling3: %s\n", e.what());
        return 2;
    }
    return 0;
}
