// basic3 (examples/basic3.cpp) with vorticity confinement pushed after the artificial viscosity: 15^3 fluid block, r = 0.05,
// DFSPH, dt = 1/200, a ground plane of boundary particles.  Prints the fluid's kinetic energy every 20 steps.
//   g++ -std=c++17 -Iinclude examples/vorticity3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o vorticity3
//   ./vorticity3 [steps] [eps]
#include <cstdio>
#include <cstdlib>

#include "salva3d_b200.hpp"

using namespace salva3d;

// examples3d/helper.rs:4-20
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

// 1/2 sum_i m_i |v_i|^2, summed in index order in double
static double kinetic_energy(const Fluid& f) {
    double s = 0.0;
    for (size_t i = 0; i < f.num_particles(); ++i) {
        const double vx = f.velocities[i].x, vy = f.velocities[i].y, vz = f.velocities[i].z;
        s += (double)f.particle_mass(i) * ((vx * vx + vy * vy) + vz * vz);
    }
    return 0.5 * s;
}

int main(int argc, char** argv) {
    const float PARTICLE_RADIUS = 0.05f, SMOOTHING_FACTOR = 2.0f;
    int steps = argc > 1 ? atoi(argv[1]) : 100;
    float eps = argc > 2 ? (float)atof(argv[2]) : 0.05f;
    try {
        LiquidWorld world(DFSPHSolver<>(), PARTICLE_RADIUS, SMOOTHING_FACTOR);
        const int n = 15;
        Fluid fluid = cube_fluid(n, n, n, PARTICLE_RADIUS, 1000.0f);
        for (auto& p : fluid.positions) p.y += 0.2f + n * PARTICLE_RADIUS;
        fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(1.0f, 0.0f));
        fluid.nonpressure_forces.push_back(std::make_shared<VorticityConfinement>(eps));
        FluidHandle fh = world.add_fluid(std::move(fluid));
        std::vector<Point3> ground;
        for (int i = -25; i <= 25; ++i)
            for (int k = -25; k <= 25; ++k) ground.push_back({i * 0.1f, 0.2f, k * 0.1f});
        world.add_boundary(Boundary(ground));
        for (int s = 1; s <= steps; ++s) {
            world.step(1.0f / 200.0f, Vector3{0.0f, -9.81f, 0.0f});
            if (s % 20 == 0) printf("vorticity3: step %d kinetic energy %.17g\n", s, kinetic_energy(world.fluids()[fh]));
        }
        printf("vorticity3: %zu particles, %d steps, eps = %g\n", world.fluids()[fh].num_particles(), steps, (double)eps);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
