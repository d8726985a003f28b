// basic3's scene (examples/basic3.cpp) run for 100 steps, then its liquid surface meshed on the device with anisotropic kernels
// (include/sph.h sph_world_extract_surface_anisotropic, default SurfaceAnisotropy): writes the mesh as an OBJ file and prints
// the vertex and triangle counts, the enclosed volume and the sum of the smoothed centres.
//   g++ -std=c++17 -Iinclude examples/surface_aniso3.cpp -Lsalva_b200 -lsalva_b200 -Wl,-rpath,$PWD/salva_b200 -o surface_aniso3
//   ./surface_aniso3 [steps = 100] [out.obj = surface_aniso3.obj]
#include <cstdio>
#include <cstdlib>

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
    const float PARTICLE_RADIUS = 0.05f, SMOOTHING_FACTOR = 2.0f;
    const int steps = argc > 1 ? atoi(argv[1]) : 100;
    const char* out = argc > 2 ? argv[2] : "surface_aniso3.obj";
    try {
        LiquidWorld world(DFSPHSolver<>(), PARTICLE_RADIUS, SMOOTHING_FACTOR);
        const int n = 15;
        Fluid fluid = cube_fluid(n, n, n, PARTICLE_RADIUS, 1000.0f);
        for (auto& p : fluid.positions) p.y += 0.2f + n * PARTICLE_RADIUS;
        fluid.nonpressure_forces.push_back(std::make_shared<ArtificialViscosity>(1.0f, 0.0f));
        const FluidHandle fh = world.add_fluid(std::move(fluid));
        std::vector<Point3> ground;
        for (int i = -25; i <= 25; ++i)
            for (int k = -25; k <= 25; ++k) ground.push_back({i * 0.1f, 0.2f, k * 0.1f});
        world.add_boundary(Boundary(ground));
        for (int s = 0; s < steps; ++s) world.step(1.0f / 200.0f, Vector3{0.0f, -9.81f, 0.0f});

        const SurfaceMesh m = world.extract_surface(SurfaceAnisotropy{}, 0.6f);
        const SurfaceEllipsoids e = world.surface_ellipsoids(fh);
        double csum = 0.0;  // the smoothed centres, summed in particle order
        for (const Point3& c : e.centres) csum += (double)c.x + (double)c.y + (double)c.z;
        double volume = 0.0;  // divergence theorem over the outward-wound triangles
        for (size_t t = 0; t < m.triangles.size(); t += 3) {
            const Point3 &a = m.vertices[m.triangles[t]], &b = m.vertices[m.triangles[t + 1]], &c = m.vertices[m.triangles[t + 2]];
            volume += ((double)a.x * ((double)b.y * c.z - (double)b.z * c.y) + (double)a.y * ((double)b.z * c.x - (double)b.x * c.z) +
                       (double)a.z * ((double)b.x * c.y - (double)b.y * c.x)) / 6.0;
        }
        FILE* f = fopen(out, "w");
        if (!f) throw std::runtime_error(std::string("cannot write ") + out);
        for (size_t v = 0; v < m.vertices.size(); ++v) fprintf(f, "v %.7g %.7g %.7g\n", m.vertices[v].x, m.vertices[v].y, m.vertices[v].z);
        for (size_t v = 0; v < m.normals.size(); ++v) fprintf(f, "vn %.7g %.7g %.7g\n", m.normals[v].x, m.normals[v].y, m.normals[v].z);
        for (size_t t = 0; t < m.triangles.size(); t += 3)
            fprintf(f, "f %u//%u %u//%u %u//%u\n", m.triangles[t] + 1, m.triangles[t] + 1, m.triangles[t + 1] + 1, m.triangles[t + 1] + 1,
                    m.triangles[t + 2] + 1, m.triangles[t + 2] + 1);
        fclose(f);
        printf("surface_aniso3: %d steps, %zu ellipsoids, centre sum %.9g, %zu vertices, %zu triangles, enclosed volume %.6f\n", steps,
               e.centres.size(), csum, m.vertices.size(), m.triangles.size() / 3, volume);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        return 2;
    }
    return 0;
}
