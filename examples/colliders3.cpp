// Rigid colliders coupled on the device, two ways (the rapier integration's ColliderCouplingSet, fluids_pipeline.rs:64-287):
// basic3.rs's ground and walls (basic3.rs:69-99) are StaticSampling colliders on a fixed body, and a ball of sample points
// on a dynamic body falls into the fluid.  The example integrates the ball itself (gravity plus the impulses the fluid
// returns through collider_impulse), standing in for the rigid-body engine.  Prints the ball's height and the impulses.
//   g++ -std=c++17 -Iinclude examples/colliders3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o colliders3
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "salva3d_b200.hpp"

using namespace salva3d;

// lattice points (spacing 2r) on the surface of an axis-aligned box of half extents he, centred at the origin
static std::vector<Point3> cuboid_samples(Vector3 he, float r) {
    std::vector<Point3> pts;
    const int nx = (int)std::lround(he.x / r), ny = (int)std::lround(he.y / r), nz = (int)std::lround(he.z / r);
    for (int i = -nx; i <= nx; i += 2)
        for (int j = -ny; j <= ny; j += 2)
            for (int k = -nz; k <= nz; k += 2)
                if (std::abs(i) >= nx - 1 || std::abs(j) >= ny - 1 || std::abs(k) >= nz - 1) pts.push_back({i * r, j * r, k * r});
    return pts;
}

static std::vector<Point3> sphere_samples(float radius, int n) {
    std::vector<Point3> pts;
    const float golden = 3.14159265f * (1.0f + std::sqrt(5.0f));
    for (int k = 0; k < n; ++k) {
        const float phi = std::acos(1.0f - 2.0f * (k + 0.5f) / n), th = golden * (k + 0.5f);
        pts.push_back({radius * std::cos(th) * std::sin(phi), radius * std::cos(phi), radius * std::sin(th) * std::sin(phi)});
    }
    return pts;
}

// R <- exp([w dt]x) R (Rodrigues), row-major
static void rotate(float* R, Vector3 w, float dt) {
    const float a = std::sqrt(w.x * w.x + w.y * w.y + w.z * w.z) * dt;
    if (a < 1e-12f) return;
    const float x = w.x * dt / a, y = w.y * dt / a, z = w.z * dt / a, c = std::cos(a), s = std::sin(a), t = 1 - c;
    const float Q[9] = {t * x * x + c, t * x * y - s * z, t * x * z + s * y, t * x * y + s * z, t * y * y + c,
                        t * y * z - s * x, t * x * z - s * y, t * y * z + s * x, t * z * z + c};
    float out[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) out[3 * i + j] = Q[3 * i] * R[j] + Q[3 * i + 1] * R[3 + j] + Q[3 * i + 2] * R[6 + j];
    std::memcpy(R, out, sizeof out);
}

int main(int argc, char** argv) {
    const float r = 0.05f, dt = 1.0f / 200.0f;
    const Vector3 g{0.0f, -9.81f, 0.0f};
    int steps = argc > 1 ? atoi(argv[1]) : 60;
    try {
        LiquidWorld world(DFSPHSolver<>(), r, 2.0f);
        std::vector<Point3> block;  // 12^3 particles resting on the ground
        for (int i = 0; i < 12; ++i)
            for (int j = 0; j < 12; ++j)
                for (int k = 0; k < 12; ++k) block.push_back({(i - 5.5f) * 2 * r, 0.25f + (j + 0.5f) * 2 * r, (k - 5.5f) * 2 * r});
        Fluid fluid(block, r, 1000.0f, InteractionGroups());
        fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(1.0f, 0.0f));
        const FluidHandle fh = world.add_fluid(std::move(fluid));

        // basic3.rs:69-99: ground cuboid (2.5, 0.2, 2.5) and four walls (0.2, 0.7, 2.5), the tank here is 1.5 wide
        struct Part { Vector3 he; Isometry3 pos; };
        const float ghw = 0.75f, ghh = 0.7f, gt = 0.2f;
        Isometry3 wall_z1, wall_z2, wall_x1, wall_x2, ground;
        const float rot_y90[9] = {0, 0, 1, 0, 1, 0, -1, 0, 0};
        std::memcpy(wall_z1.rotation, rot_y90, sizeof rot_y90);
        std::memcpy(wall_z2.rotation, rot_y90, sizeof rot_y90);
        wall_z1.translation = {0, ghh, ghw + gt};
        wall_z2.translation = {0, ghh, -ghw - gt};
        wall_x1.translation = {ghw + gt, ghh, 0};
        wall_x2.translation = {-ghw - gt, ghh, 0};
        ground.translation = {0, 0, 0};
        const Part tank[5] = {{{gt, ghh, ghw + gt}, wall_z1}, {{gt, ghh, ghw + gt}, wall_z2}, {{gt, ghh, ghw}, wall_x1},
                              {{gt, ghh, ghw}, wall_x2}, {{ghw + 2 * gt, gt, ghw + 2 * gt}, ground}};
        size_t n_tank = 0;
        for (const Part& p : tank) {
            std::vector<Point3> samples = cuboid_samples(p.he, r);
            n_tank += samples.size();
            const ColliderHandle c = world.register_coupling(world.add_boundary(Boundary({})), ColliderSampling::StaticSampling(std::move(samples)));
            world.set_collider_state(c, p.pos, SPH_BODY_FIXED);
        }

        // the ball: a dynamic body the example integrates
        const float radius = 0.25f, density = 500.0f;
        const float mass = density * 4.0f / 3.0f * 3.14159265f * radius * radius * radius, inertia = 0.4f * mass * radius * radius;
        const ColliderHandle ball = world.register_coupling(world.add_boundary(Boundary({})), ColliderSampling::StaticSampling(sphere_samples(radius, 400)));
        Isometry3 pose;
        pose.translation = {0.1f, 1.9f, 0.0f};
        Vector3 v{0.0f, -3.0f, 0.0f}, w{0.0f, 0.0f, 0.0f};
        float max_impulse = 0.0f, min_y = pose.translation.y;
        for (int s = 0; s < steps; ++s) {
            world.set_collider_state(ball, pose, SPH_BODY_DYNAMIC, v, w, pose.translation);
            world.step(dt, g);
            const auto imp = world.collider_impulse(ball);  // transmit_forces: apply_impulse_at_point
            const Vector3 lin = imp.first, ang = imp.second;
            max_impulse = std::fmax(max_impulse, std::sqrt(lin.x * lin.x + lin.y * lin.y + lin.z * lin.z));
            v = {v.x + g.x * dt + lin.x / mass, v.y + g.y * dt + lin.y / mass, v.z + g.z * dt + lin.z / mass};
            w = {w.x + ang.x / inertia, w.y + ang.y / inertia, w.z + ang.z / inertia};
            pose.translation = {pose.translation.x + v.x * dt, pose.translation.y + v.y * dt, pose.translation.z + v.z * dt};
            rotate(pose.rotation, w, dt);
            min_y = std::fmin(min_y, pose.translation.y);
        }
        const Fluid& f = world.fluids()[fh];
        printf("colliders3: %zu particles, %zu tank samples, %d steps, ball y = %.4f (lowest %.4f), vy = %.4f, max |impulse| = %.6g\n", f.num_particles(),
               n_tank, steps, pose.translation.y, min_y, v.y, max_impulse);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
