// Cylinder and cone colliders coupled by DynamicContactSampling: a 10 x 8 x 10 block of fluid poured onto a fixed cone
// (apex up) and a cylinder lying on its side on a dynamic body, inside an open tank sampled as a static boundary.  Every step
// both shapes sample the surface under the nearby fluid and push penetrating particles out; the cylinder's body reads back
// the impulse the fluid applied to it.
// Prints the bookkeeping: the first step with samples on each shape, the steps without samples after it, non-finite values,
// the deepest fluid particle inside either solid at the end, and the cylinder's last impulse.
//   g++ -std=c++17 -Iinclude examples/cylinder_cone3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o cylinder_cone3
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "salva3d_b200.hpp"

using namespace salva3d;

// depth of p inside a solid of revolution posed at t with the identity (cone) or a quarter turn about z (cylinder, axis
// along world x); <= 0 outside.  The cone's apex is at +a along its axis.
static double depth_inside(bool cone, const Point3& p, const Point3& t, double a, double r) {
    double y, rho;
    if (cone) {
        y = p.y - t.y;
        rho = std::hypot(p.x - t.x, p.z - t.z);
    } else {
        y = p.x - t.x;
        rho = std::hypot(p.y - t.y, p.z - t.z);
    }
    if (!cone) return std::min(r - rho, a - std::fabs(y));
    const double L = std::hypot(r, 2 * a);
    return std::min(y + a, (r * (a - y) - 2 * a * rho) / L);
}

int main(int argc, char** argv) {
    const float R = 0.025f, dt = 1.0f / 200.0f;
    const int steps = argc > 1 ? atoi(argv[1]) : 300;
    try {
        LiquidWorld world(DFSPHSolver<>(), R, 2.0f);
        std::vector<Point3> block;
        for (int i = 0; i < 10; ++i)
            for (int j = 0; j < 8; ++j)
                for (int k = 0; k < 10; ++k) block.push_back({0.3f + (i + 0.5f) * 2 * R, 0.55f + (j + 0.5f) * 2 * R, 0.3f + (k + 0.5f) * 2 * R});
        Fluid fluid(block, R, 1000.0f, InteractionGroups());
        fluid.nonpressure_forces.push_back(std::make_shared<XSPHViscosity>(0.5f, 0.0f));
        const FluidHandle fh = world.add_fluid(std::move(fluid));

        // an open tank [0, 1.2] x [0, 0.8] x [0, 1.2], its floor and walls sampled at spacing 2R
        std::vector<Point3> tank;
        const int n = 24;
        for (int i = 0; i <= n; ++i)
            for (int k = 0; k <= n; ++k) tank.push_back({i * 2 * R, 0.0f, k * 2 * R});
        for (int i = 0; i <= n; ++i)
            for (int j = 1; j <= 16; ++j) {
                tank.push_back({i * 2 * R, j * 2 * R, 0.0f});
                tank.push_back({i * 2 * R, j * 2 * R, n * 2 * R});
                tank.push_back({0.0f, j * 2 * R, i * 2 * R});
                tank.push_back({n * 2 * R, j * 2 * R, i * 2 * R});
            }
        world.add_boundary(Boundary(tank));

        const Cone cone{0.12f, 0.15f};          // apex up, base on the floor
        const Cylinder cyl{0.15f, 0.06f};       // axis along world x after a quarter turn about z
        const Point3 tc{0.45f, 0.12f, 0.45f}, ty{0.75f, 0.06f, 0.65f};
        const BoundaryHandle bc = world.add_boundary(Boundary({}));
        const BoundaryHandle by = world.add_boundary(Boundary({}));
        const ColliderHandle cc = world.register_coupling(bc, ColliderSampling::DynamicContactSampling(cone));
        const ColliderHandle cy = world.register_coupling(by, ColliderSampling::DynamicContactSampling(cyl));
        Isometry3 pc, py;
        pc.translation = tc;
        py.translation = ty;
        const Real quarter[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1};
        std::copy(quarter, quarter + 9, py.rotation);
        world.set_collider_state(cc, pc, SPH_BODY_FIXED);
        world.set_collider_state(cy, py, SPH_BODY_DYNAMIC, Vector3(), Vector3(), ty);

        int first[2] = {-1, -1};
        size_t before[2] = {0, 0}, empty[2] = {0, 0};
        std::pair<Vector3, Vector3> imp;
        for (int s = 0; s < steps; ++s) {
            world.step(dt, Vector3{0.0f, -9.81f, 0.0f});
            const size_t ns[2] = {world.boundaries()[bc].num_particles(), world.boundaries()[by].num_particles()};
            for (int q = 0; q < 2; ++q) {
                if (first[q] < 0 && ns[q]) first[q] = s;
                if (first[q] < 0) before[q] += ns[q];
                else if (!ns[q]) ++empty[q];
            }
            imp = world.collider_impulse(cy);
        }
        const Fluid& f = world.fluids()[fh];
        size_t nan = 0;
        double deepest = -1e30;
        for (const auto& p : f.positions) {
            if (!(std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z))) {
                ++nan;
                continue;
            }
            deepest = std::max({deepest, depth_inside(true, p, tc, cone.half_height, cone.radius), depth_inside(false, p, ty, cyl.half_height, cyl.radius)});
        }
        printf("cylinder_cone3: %zu particles, %d steps, first samples at steps %d and %d, %zu and %zu samples before, %zu and %zu empty "
               "steps after, %zu non-finite, deepest particle %.5f inside, cylinder impulse (%.5g, %.5g, %.5g)\n",
               f.num_particles(), steps, first[0], first[1], before[0], before[1], empty[0], empty[1], nan, deepest, imp.first.x, imp.first.y,
               imp.first.z);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
