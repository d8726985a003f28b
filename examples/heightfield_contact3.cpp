// examples3d/heightfield3.rs:19-93 with the ground coupled by DynamicContactSampling instead of StaticSampling: a 15^3
// block of fluid thrown at 10 m/s onto parry's HeightField (41 x 41 heights, scale (12, 1, 12)) on a fixed body.  Every step
// the ground samples its closest surface points under the nearby fluid.  parry's heightfield point query never reports a
// point as inside, so the ground never pushes fluid out: the samples' pressure alone holds the fluid up.
// Prints the bookkeeping: the first step with ground samples, the range of the sample count from then on, non-finite
// values, and the deepest fluid particle below the triangulated surface.
//   g++ -std=c++17 -Iinclude examples/heightfield_contact3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o heightfield_contact3
#include <algorithm>
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

// height of the triangulated surface at (x, z) over the footprint (DESIGN.md section 11), in double
static double surface_height(const HeightField& g, double x, double z) {
    const double dx = g.scale.x / (g.ncols - 1.0), dz = g.scale.z / (g.nrows - 1.0);
    const double u = std::min(std::max((x + g.scale.x / 2) / dx, 0.0), g.ncols - 1.000001);
    const double v = std::min(std::max((z + g.scale.z / 2) / dz, 0.0), g.nrows - 1.000001);
    const int j = (int)u, i = (int)v;
    const double fu = u - j, fv = v - i;
    auto h = [&](int r, int c) { return (double)g.heights[(size_t)r * g.ncols + c]; };
    const double y = fu + fv <= 1.0 ? h(i, j) + fu * (h(i, j + 1) - h(i, j)) + fv * (h(i + 1, j) - h(i, j))
                                    : h(i + 1, j + 1) + (1 - fu) * (h(i + 1, j) - h(i + 1, j + 1)) + (1 - fv) * (h(i, j + 1) - h(i + 1, j + 1));
    return y * g.scale.y;
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

        // heightfield3.rs:46-61: 3.0 on the rim, sin(i * 12 / 40) + cos(j * 12 / 40) inside
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
        const BoundaryHandle bh = world.add_boundary(Boundary({}));
        const ColliderHandle c = world.register_coupling(bh, ColliderSampling::DynamicContactSampling(ground));
        world.set_collider_state(c, Isometry3(), SPH_BODY_FIXED);  // RigidBodyBuilder::fixed()

        // the block starts above the ground's reach: count the steps from its first contact on
        size_t smin = (size_t)-1, smax = 0, empty_steps = 0;
        int first = -1;
        for (int s = 0; s < steps; ++s) {
            world.step(dt, Vector3{0.0f, -9.81f, 0.0f});
            const size_t ns = world.boundaries()[bh].num_particles();
            if (first < 0 && ns) first = s;
            if (first < 0) continue;
            smin = std::min(smin, ns);
            smax = std::max(smax, ns);
            if (ns == 0) ++empty_steps;
        }
        const Fluid& f = world.fluids()[fh];
        size_t nan = 0;
        double deepest = -1e30;
        for (const auto& p : f.positions) {
            if (!(std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z))) {
                ++nan;
                continue;
            }
            if (std::fabs(p.x) <= 6.0f && std::fabs(p.z) <= 6.0f) deepest = std::max(deepest, surface_height(ground, p.x, p.z) - p.y);
        }
        printf("heightfield_contact3: %zu particles, %d steps, first contact at step %d, ground samples per step %zu..%zu, "
               "%zu steps without samples since, %zu non-finite, deepest particle %.4f below the surface\n",
               f.num_particles(), steps, first, first < 0 ? (size_t)0 : smin, smax, empty_steps, nan, deepest);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
