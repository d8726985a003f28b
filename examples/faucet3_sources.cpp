// examples3d/faucet3.rs (faucet3.rs:19-137) with the per-step callback (faucet3.rs:69-105) replaced by a particle source and
// sink that the engine applies on the device at the start of every step: a 10 x 10 sheet every 12 steps (0.06 s at
// dt = 1 / 200) and the removal of every particle below y = -2.  With --host the same rule runs through fluids_mut()
// (delete_particle_at_next_timestep, add_particles) before each step, as faucet3 does; both modes print the same line.
//   g++ -std=c++17 -Iinclude examples/faucet3_sources.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o faucet3_sources
//   ./faucet3_sources [steps] [--host]
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>

#include "salva3d_b200.hpp"

using namespace salva3d;

// the ball of faucet3.rs:51-65, sampled on its surface at spacing ~2r (as examples/faucet3.cpp)
static std::vector<Point3> ball_surface(Real radius, Real particle_rad) {
    const double pi = 3.14159265358979323846;
    const int n = (int)std::ceil(4.0 * pi * radius * radius / (4.0 * particle_rad * particle_rad));
    std::vector<Point3> pts;
    const double golden = pi * (3.0 - std::sqrt(5.0));
    for (int i = 0; i < n; ++i) {
        const double y = 1.0 - 2.0 * (i + 0.5) / n, rho = std::sqrt(1.0 - y * y), th = golden * i;
        pts.push_back({(Real)(radius * rho * std::cos(th)), (Real)(radius * y), (Real)(radius * rho * std::sin(th))});
    }
    return pts;
}

int main(int argc, char** argv) {
    const Real PARTICLE_RADIUS = 0.025f / 2.0f, SMOOTHING_FACTOR = 2.0f, dt = 1.0f / 200.0f, FLOOR = -2.0f;
    const uint32_t INTERVAL = 12;
    int steps = 400;
    bool host = false;
    for (int a = 1; a < argc; ++a) {
        if (!std::strcmp(argv[a], "--host")) host = true;
        else steps = std::atoi(argv[a]);
    }
    try {
        LiquidWorld world(DFSPHSolver<>(), PARTICLE_RADIUS, SMOOTHING_FACTOR);
        Fluid fluid({}, PARTICLE_RADIUS, 1000.0f, InteractionGroups());  // faucet3.rs:40-45: no particle yet
        fluid.nonpressure_forces.push_back(std::make_shared<XSPHViscosity>(0.5f, 0.0f));
        fluid.nonpressure_forces.push_back(std::make_shared<Akinci2013SurfaceTension>(1.0f, 10.0f));
        const FluidHandle fh = world.add_fluid(std::move(fluid));
        world.add_boundary(Boundary(ball_surface(0.15f, PARTICLE_RADIUS)));
        // the sheet of faucet3.rs:88-103
        const Real height = 0.6f, diam = PARTICLE_RADIUS * 2.0f;
        const int nside = 10;
        const Real shift = -nside * PARTICLE_RADIUS;
        std::vector<Point3> sheet;
        std::vector<Vector3> sheet_vel;
        for (int i = 0; i < nside; ++i)
            for (int j = 0; j < nside; ++j) {
                sheet.push_back({i * diam + shift, height, j * diam + shift});
                sheet_vel.push_back(Vector3{0.0f, 0.0f, 0.0f});
            }
        if (!host) {
            const Real inf = std::numeric_limits<Real>::infinity();
            world.add_particle_sink(fh, Vector3{-inf, -inf, -inf}, Vector3{inf, FLOOR, inf});  // faucet3.rs:77-81: y < -2
            world.add_particle_source(fh, sheet, &sheet_vel, INTERVAL);
        }
        size_t emitted = 0, removed = 0;
        for (int s = 0; s < steps; ++s) {
            if (host) {
                Fluid& f = world.fluids_mut()[fh];
                const Real inf = std::numeric_limits<Real>::infinity();
                for (size_t i = 0; i < f.num_particles(); ++i) {
                    const Point3& p = f.positions[i];  // the sink's box test: lo <= x < hi on every axis
                    if (-inf <= p.x && p.x < inf && -inf <= p.y && p.y < FLOOR && -inf <= p.z && p.z < inf) {
                        f.delete_particle_at_next_timestep(i);
                        ++removed;
                    }
                }
                if (s % INTERVAL == 0) {
                    f.add_particles(sheet, &sheet_vel);
                    emitted += sheet.size();
                }
            }
            world.step(dt, Vector3{0.0f, -9.81f, 0.0f});
            if (!host) {
                const std::pair<uint32_t, uint32_t> e = world.step_edits(fh);
                removed += e.first;
                emitted += e.second;
            }
        }
        const Fluid& f = world.fluids()[fh];
        double checksum = 0.0;
        for (size_t i = 0; i < f.num_particles(); ++i) checksum += (i + 1) * ((double)f.positions[i].x + 2.0 * f.positions[i].y + 3.0 * f.positions[i].z);
        std::printf("faucet3_sources: %d steps, emitted %zu, removed %zu, alive %zu, checksum %.9e\n", steps, emitted, removed, f.num_particles(), checksum);
        if (f.num_particles() + removed != emitted) {
            std::fprintf(stderr, "faucet3_sources: particle bookkeeping does not add up\n");
            return 1;
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "faucet3_sources: %s\n", e.what());
        return 2;
    }
    return 0;
}
