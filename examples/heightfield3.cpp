// examples3d/heightfield3.rs:19-93: a 15^3 block of fluid thrown at 10 m/s onto a heightfield ground.  The ground is
// parry's HeightField (41 x 41 heights, scale (12, 1, 12)), surface-sampled on the device at r / 1.5 with
// salva3d::sampling::shape_surface_ray_sample and coupled as a StaticSampling collider on a fixed body.
// Prints the bookkeeping; `heightfield3 STEPS DUMP` also writes the heights, the ground samples and the final fluid
// positions to DUMP (raw float32: heights, then sample count and xyz, then particle count and xyz).
//   g++ -std=c++17 -Iinclude examples/heightfield3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o heightfield3
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "salva3d_b200.hpp"

using namespace salva3d;

static std::vector<Point3> cube_fluid(int ni, int nj, int nk, float particle_rad) {  // helper.rs:4-20
    std::vector<Point3> points;
    const float hx = ni * particle_rad, hy = nj * particle_rad, hz = nk * particle_rad;
    for (int i = 0; i < ni; ++i)
        for (int j = 0; j < nj; ++j)
            for (int k = 0; k < nk; ++k)
                points.push_back({i * particle_rad * 2.0f + particle_rad - hx, j * particle_rad * 2.0f + particle_rad - hy,
                                  k * particle_rad * 2.0f + particle_rad - hz});
    return points;
}

static void dump_floats(FILE* f, const void* p, size_t n) {
    if (n && fwrite(p, sizeof(float), n, f) != n) throw std::runtime_error("short write");
}

int main(int argc, char** argv) {
    const float PARTICLE_RADIUS = 0.15f, SMOOTHING_FACTOR = 2.0f, dt = 1.0f / 200.0f;
    const int steps = argc > 1 ? atoi(argv[1]) : 200;
    try {
        LiquidWorld world(DFSPHSolver<>(), PARTICLE_RADIUS, SMOOTHING_FACTOR);
        const int nparticles = 15;
        std::vector<Point3> block = cube_fluid(nparticles, nparticles, nparticles, PARTICLE_RADIUS);
        const float ty = 1.0f + nparticles * PARTICLE_RADIUS * 2.0f;  // heightfield3.rs:33-37
        for (auto& p : block) p.y += ty;
        Fluid fluid(block, PARTICLE_RADIUS, 1000.0f, InteractionGroups());
        fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(1.0f, 0.0f));
        fluid.velocities.assign(fluid.positions.size(), Vector3{0.0f, -10.0f, 0.0f});  // :40
        const FluidHandle fh = world.add_fluid(std::move(fluid));

        // heightfield3.rs:46-61: DMatrix::from_fn(i, j), 3.0 on the rim, sin(i * 12 / 40) + cos(j * 12 / 40) inside
        const int nsubdivs = 40;
        HeightField ground;
        ground.nrows = ground.ncols = nsubdivs + 1;
        ground.scale = {12.0f, 1.0f, 12.0f};
        ground.heights.resize((size_t)ground.nrows * ground.ncols);
        for (int i = 0; i <= nsubdivs; ++i)
            for (int j = 0; j <= nsubdivs; ++j) {
                const float x = i * ground.scale.x / (float)nsubdivs, z = j * ground.scale.z / (float)nsubdivs;
                ground.heights[(size_t)i * ground.ncols + j] = (i == 0 || i == nsubdivs || j == 0 || j == nsubdivs) ? 3.0f : std::sin(x) + std::cos(z);
            }
        std::vector<Point3> samples = sampling::shape_surface_ray_sample(world, ground, PARTICLE_RADIUS / 1.5f);  // :68-70
        const size_t n_samples = samples.size();
        const BoundaryHandle bh = world.add_boundary(Boundary({}));
        const ColliderHandle c = world.register_coupling(bh, ColliderSampling::StaticSampling(samples));
        world.set_collider_state(c, Isometry3(), SPH_BODY_FIXED);  // RigidBodyBuilder::fixed()

        for (int s = 0; s < steps; ++s) world.step(dt, Vector3{0.0f, -9.81f, 0.0f});
        const Fluid& f = world.fluids()[fh];
        size_t nan = 0;
        float ymin = 1e30f;
        for (const auto& p : f.positions) {
            if (!(std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z))) ++nan;
            else ymin = std::fmin(ymin, p.y);
        }
        printf("heightfield3: %zu particles, %zu ground samples, boundary holds %zu, %d steps, %zu non-finite, lowest y = %.4f\n",
               f.num_particles(), n_samples, world.boundaries()[bh].num_particles(), steps, nan, ymin);
        if (argc > 2) {
            FILE* out = fopen(argv[2], "wb");
            if (!out) throw std::runtime_error("cannot open the dump file");
            dump_floats(out, ground.heights.data(), ground.heights.size());
            const float ns = (float)n_samples, np = (float)f.num_particles();
            dump_floats(out, &ns, 1);
            dump_floats(out, samples.data(), 3 * n_samples);
            dump_floats(out, &np, 1);
            dump_floats(out, f.positions.data(), 3 * f.positions.size());
            fclose(out);
        }
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
