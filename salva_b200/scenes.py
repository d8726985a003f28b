"""Deterministic synthetic scenes for the salva3d step path (SURVEY.md §8(d)).

All generators are pure numpy/f32 and produce the same bytes on every machine, so the
oracle and the CUDA engine are always driven with identical inputs.

  cube_fluid          restates examples3d/helper.rs:4-20 (the reference's own block generator)
  jitter              splitmix64 jitter in [-0.05r, 0.05r)^3 (removes the marginal d == h lattice pairs)
  cuboid_surface      deterministic stand-in for sampling::shape_surface_ray_sample on a cuboid
                      (ray_sampling.rs:9-15 is out of scope: parry ray casts, HashSet order)
  open_tank           single-layer lattice on 5 faces of an open-top box
  scene_c1..scene_c5  the BASELINE.json configs
"""
import numpy as np

F32 = np.float32
GRAVITY = (0.0, -9.81, 0.0)

# force kinds (include/sph.h SPH_FORCE_*)
XSPH, ARTIFICIAL, AKINCI2013, BECKER2009, HE2014, WCSPH, DFSPH_VISCOSITY, VORTICITY = 0, 1, 2, 3, 4, 5, 6, 7
DFSPH, IISPH = 0, 1


def xsph_viscosity(fluid_coeff, boundary_coeff=0.0):
    """XSPHViscosity::new(fluid, boundary)  xsph_viscosity.rs:19-26"""
    return (XSPH, [fluid_coeff, boundary_coeff])


def artificial_viscosity(fluid_coeff, boundary_coeff=0.0, alpha=1.0, beta=0.0, speed_of_sound=10.0):
    """ArtificialViscosity::new(fluid, boundary)  artificial_viscosity.rs:27-38 (alpha=1, beta=0, c=10)"""
    return (ARTIFICIAL, [fluid_coeff, boundary_coeff, alpha, beta, speed_of_sound])


def akinci2013_surface_tension(tension, adhesion=0.0):
    """Akinci2013SurfaceTension::new(tension, adhesion)  akinci2013_surface_tension.rs:27-35"""
    return (AKINCI2013, [tension, adhesion])


def becker2009_elasticity(young, poisson, nonlinear=True):
    """Becker2009Elasticity::new(E, nu, nonlinear)  becker2009_elasticity.rs:60-76"""
    return (BECKER2009, [young, poisson, 1.0 if nonlinear else 0.0])


def he2014_surface_tension(fluid_tension, boundary_tension=0.0):
    """He2014SurfaceTension::new(fluid, boundary)  he2014_surface_tension.rs:21-29"""
    return (HE2014, [fluid_tension, boundary_tension])


def wcsph_surface_tension(fluid_tension, boundary_tension=0.0):
    """WCSPHSurfaceTension::new(fluid, boundary)  wcsph_surface_tension.rs:21-27 (boundary term: see include/sph.h)"""
    return (WCSPH, [fluid_tension, boundary_tension])


def dfsph_viscosity(viscosity_coefficient, min_viscosity_iter=1, max_viscosity_iter=50, max_viscosity_error=0.01):
    """DFSPHViscosity::new(coefficient) + public tunables  dfsph_viscosity.rs:86-124"""
    return (DFSPH_VISCOSITY, [viscosity_coefficient, float(min_viscosity_iter), float(max_viscosity_iter), max_viscosity_error])


def vorticity_confinement(eps):
    """Vorticity confinement with strength eps > 0 in m/s (include/sph.h SPH_FORCE_VORTICITY_CONFINEMENT; no reference counterpart)"""
    return (VORTICITY, [eps])


def cube_fluid(ni, nj, nk, particle_rad):
    """examples3d/helper.rs:4-20, f32 arithmetic in the same order (i slowest, k fastest)."""
    r = F32(particle_rad)
    two = F32(2.0)
    i = np.arange(ni, dtype=F32)[:, None, None]
    j = np.arange(nj, dtype=F32)[None, :, None]
    k = np.arange(nk, dtype=F32)[None, None, :]
    half = np.array([ni, nj, nk], dtype=F32) * r
    x = np.broadcast_to(i * r * two + r - half[0], (ni, nj, nk))
    y = np.broadcast_to(j * r * two + r - half[1], (ni, nj, nk))
    z = np.broadcast_to(k * r * two + r - half[2], (ni, nj, nk))
    return np.stack([x, y, z], axis=-1).reshape(-1, 3).astype(F32)


def _splitmix64(seed, n, start=0):
    with np.errstate(over="ignore"):
        k = np.arange(start + 1, start + n + 1, dtype=np.uint64)
        z = np.uint64(seed) + k * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def jitter(points, particle_rad, seed, amplitude=0.05, first_index=0):
    """delta in [-amplitude*r, amplitude*r)^3 from splitmix64(seed) in particle-index order; `first_index` is the
    global index of points[0] (a rank that generates only its slab of a block gets the same bytes as the whole block)."""
    n = len(points)
    u = (_splitmix64(seed, 3 * n, 3 * first_index) >> np.uint64(40)).astype(F32) * F32(1.0 / (1 << 24))  # [0,1)
    d = (u * F32(2.0) - F32(1.0)) * F32(amplitude) * F32(particle_rad)
    return (points + d.reshape(n, 3)).astype(F32)


def _face(axis, coord, lo, hi, spacing):
    """Lattice of `spacing` covering [lo, hi] in the two in-plane axes at `coord` on `axis`."""
    a, b = [d for d in range(3) if d != axis]
    na = int(np.floor((hi[a] - lo[a]) / spacing + 1e-4)) + 1
    nb = int(np.floor((hi[b] - lo[b]) / spacing + 1e-4)) + 1
    ua = F32(lo[a]) + np.arange(na, dtype=F32) * F32(spacing)
    ub = F32(lo[b]) + np.arange(nb, dtype=F32) * F32(spacing)
    pts = np.empty((na, nb, 3), F32)
    pts[..., axis] = F32(coord)
    pts[..., a] = ua[:, None]
    pts[..., b] = ub[None, :]
    return pts.reshape(-1, 3)


def cuboid_surface(half_extents, particle_rad, center=(0.0, 0.0, 0.0)):
    """Surface lattice (spacing 2r) of an axis-aligned cuboid, edges/corners not duplicated."""
    he = np.asarray(half_extents, dtype=np.float64)
    s = 2.0 * particle_rad
    lo, hi = -he, he
    faces = []
    # +-y faces cover the full rectangle; +-x faces skip the y extremes; +-z skip x and y extremes.
    faces.append(_face(1, lo[1], lo, hi, s))
    faces.append(_face(1, hi[1], lo, hi, s))
    lo_y, hi_y = lo.copy(), hi.copy()
    lo_y[1] += s
    hi_y[1] -= s
    faces.append(_face(0, lo[0], lo_y, hi_y, s))
    faces.append(_face(0, hi[0], lo_y, hi_y, s))
    lo_xy, hi_xy = lo_y.copy(), hi_y.copy()
    lo_xy[0] += s
    hi_xy[0] -= s
    faces.append(_face(2, lo[2], lo_xy, hi_xy, s))
    faces.append(_face(2, hi[2], lo_xy, hi_xy, s))
    pts = np.concatenate(faces, axis=0)
    return (pts + np.asarray(center, F32)).astype(F32)


def open_tank(lo, hi, particle_rad):
    """Single-layer lattice (spacing 2r) on the floor and 4 walls of the box [lo, hi]; top open.

    lo/hi are the coordinates of the boundary-particle planes themselves.
    """
    lo = np.asarray(lo, np.float64)
    hi = np.asarray(hi, np.float64)
    s = 2.0 * particle_rad
    faces = [_face(1, lo[1], lo, hi, s)]  # floor
    lo_w, hi_w = lo.copy(), hi.copy()
    lo_w[1] += s
    faces.append(_face(0, lo[0], lo_w, hi_w, s))
    faces.append(_face(0, hi[0], lo_w, hi_w, s))
    lo_z, hi_z = lo_w.copy(), hi_w.copy()
    lo_z[0] += s
    hi_z[0] -= s
    faces.append(_face(2, lo[2], lo_z, hi_z, s))
    faces.append(_face(2, hi[2], lo_z, hi_z, s))
    return np.concatenate(faces, axis=0).astype(F32)


def block_lattice(nx, ny, nz, particle_rad, origin=(0.0, 0.0, 0.0)):
    """Lattice block with min corner at `origin`: centres at origin + (i+0.5)*2r, x slowest, z fastest."""
    r = F32(particle_rad)
    o = np.asarray(origin, F32)
    x = o[0] + (np.arange(nx, dtype=F32) * F32(2.0) + F32(1.0)) * r
    y = o[1] + (np.arange(ny, dtype=F32) * F32(2.0) + F32(1.0)) * r
    z = o[2] + (np.arange(nz, dtype=F32) * F32(2.0) + F32(1.0)) * r
    pts = np.empty((nx, ny, nz, 3), F32)
    pts[..., 0] = x[:, None, None]
    pts[..., 1] = y[None, :, None]
    pts[..., 2] = z[None, None, :]
    return pts.reshape(-1, 3)


def _dam_break(nx, ny, nz, r, dt, forces, solver=DFSPH, name="", tank_x_factor=2.0, jitter_seed=0x5A17A, compress=1.0, amplitude=0.05,
               x_range=None):
    """Block of nx*ny*nz particles (lattice spacing 2r*compress, jittered) in an open tank.  compress < 1 starts the block
    over-dense (0.93 ~ rest density, 0.90 ~ +10 %: the Jacobi loops run several iterations from the first step).
    x_range = (i0, i1) generates only the lattice planes i0 <= i < i1 (the slab of one rank) with the same bytes."""
    s = 2.0 * r
    if x_range is None:
        pts = jitter(block_lattice(nx, ny, nz, r * compress), r, jitter_seed, amplitude=amplitude)
    else:
        i0, i1 = x_range
        # same f32 arithmetic as block_lattice: x = (2 i + 1) * r for the global lattice index i
        rr = F32(r * compress)
        x = (np.arange(i0, i1, dtype=F32) * F32(2.0) + F32(1.0)) * rr
        y = (np.arange(ny, dtype=F32) * F32(2.0) + F32(1.0)) * rr
        z = (np.arange(nz, dtype=F32) * F32(2.0) + F32(1.0)) * rr
        blk = np.empty((i1 - i0, ny, nz, 3), F32)
        blk[..., 0] = x[:, None, None]
        blk[..., 1] = y[None, :, None]
        blk[..., 2] = z[None, None, :]
        blk = blk.reshape(-1, 3)
        pts = jitter(blk, r, jitter_seed, amplitude=amplitude, first_index=i0 * ny * nz)
    lo = (-r, -r, -r)
    hi = (nx * s * tank_x_factor + r, ny * s + 4 * s + r, nz * s + r)
    # snap hi to the lattice so walls sit exactly one spacing outside the block in z
    tank = open_tank(lo, hi, r)
    return dict(name=name, particle_radius=r, smoothing_factor=2.0, dt=dt, gravity=GRAVITY, solver=solver,
                fluids=[dict(positions=pts, density0=1000.0, forces=forces)],
                boundaries=[dict(positions=tank)])


def scene_c1():
    """examples3d/basic3.rs:16-118: 15^3 block, r=0.05, dt=1/200, DFSPH + ArtificialViscosity(1,0);
    ground cuboid (2.5,0.2,2.5) + 4 walls (0.2,0.7,2.5), each its own Boundary. No jitter."""
    r = 0.05
    n = 15
    pts = cube_fluid(n, n, n, r)
    pts = (pts + np.array([0.0, F32(0.2) + F32(n) * F32(r), 0.0], F32)).astype(F32)
    gt, ghw, ghh = 0.2, 2.5, 0.7
    wall = cuboid_surface((gt, ghh, ghw), r)
    # Isometry3::new(t, y * pi/2): rotate about y by 90deg: (x,y,z) -> (z, y, -x)
    rot = np.stack([wall[:, 2], wall[:, 1], -wall[:, 0]], axis=1).astype(F32)
    bounds = [dict(positions=(rot + np.array([0.0, ghh, ghw], F32)).astype(F32)),
              dict(positions=(rot + np.array([0.0, ghh, -ghw], F32)).astype(F32)),
              dict(positions=(wall + np.array([ghw, ghh, 0.0], F32)).astype(F32)),
              dict(positions=(wall + np.array([-ghw, ghh, 0.0], F32)).astype(F32)),
              dict(positions=cuboid_surface((ghw, gt, ghw), r))]
    return dict(name="C1-basic3", particle_radius=r, smoothing_factor=2.0, dt=1.0 / 200.0, gravity=GRAVITY,
                solver=DFSPH, fluids=[dict(positions=pts, density0=1000.0, forces=[artificial_viscosity(1.0, 0.0)])],
                boundaries=bounds)


def scene_tension_small():
    """Not a reference config: a small jittered, slightly compressed block in an open tank with the two surface-tension
    rows added in §8(f).3 (He2014 incl. its boundary reaction, WCSPH fluid term) — used for a committed golden fixture."""
    r = 0.05
    nx, ny, nz = 10, 8, 7
    pts = jitter(block_lattice(nx, ny, nz, r * 0.95), r, 71, amplitude=0.3)
    tank = open_tank((-r, -r, -r), (nx * 2 * r + r, 1.0, nz * 2 * r + r), r)
    return dict(name="tension-small", particle_radius=r, smoothing_factor=2.0, dt=0.004, gravity=GRAVITY, solver=DFSPH,
                fluids=[dict(positions=pts, density0=1000.0, forces=[he2014_surface_tension(40.0, 30.0), wcsph_surface_tension(2.0)])],
                boundaries=[dict(positions=tank, want_forces=True)])


def scene_c2(n=100, **kw):
    """1M-particle cube dam-break, DFSPH + XSPHViscosity(0.5, 0), r=0.025, dt=1/1000."""
    return _dam_break(n, n, n, 0.025, 1.0 / 1000.0, [xsph_viscosity(0.5, 0.0)], name="C2-dam-%d" % (n ** 3), **kw)


def scene_c3(n=216, **kw):
    """10M particles, DFSPH + Akinci2013SurfaceTension(1, 0) (roofline capture config)."""
    return _dam_break(n, n, n, 0.025, 1.0 / 1000.0, [akinci2013_surface_tension(1.0, 0.0)],
                      name="C3-dam-%d" % (n ** 3), **kw)


def scene_c4(nx=512, ny=250, nz=250, **kw):
    """32M particles DFSPH (no extra force), long axis = slab axis x."""
    return _dam_break(nx, ny, nz, 0.025, 1.0 / 1000.0, [], name="C4-dam-%d" % (nx * ny * nz), tank_x_factor=1.25, **kw)


def slab_scene(scene_fn, rank, nranks, nx, **kw):
    """Rank `rank`'s slab of a dam-break scene whose block is nx lattice planes long in x, generated WITHOUT building the
    other ranks' particles.  Lattice plane i sits at x_i = (2 i + 1) r c (c = `compress`, jitter < amplitude * r on top); the
    cut before plane i is legal when a cell boundary k*h (h = 4 r) separates planes i-1 and i with the jitter margin, so
    that both sides own whole cell columns.  The cuts are the legal ones closest to an even split.  Returns the partitioned
    scene dict that salva_b200.slab.populate_slab() accepts (fluids carry global ids, `slab` = owned cell columns)."""
    probe = scene_fn(x_range=(0, 0), **kw)
    r = float(probe["particle_radius"])
    c = float(kw.get("compress", 1.0))
    amp = float(kw.get("amplitude", 0.05)) * r
    h = np.float32(r) * np.float32(probe["smoothing_factor"]) * np.float32(2.0)
    rr = F32(r * c)
    x = ((np.arange(nx, dtype=F32) * F32(2.0) + F32(1.0)) * rr).astype(np.float64)   # same f32 arithmetic as the generator
    col_hi_prev = np.floor((x[:-1] + amp * 1.001) / float(h))   # largest column plane i-1 can reach
    col_lo_next = np.floor((x[1:] - amp * 1.001) / float(h))    # smallest column plane i can reach
    legal = np.nonzero(col_lo_next > col_hi_prev)[0] + 1        # cut before plane i
    cuts = [0]
    for k in range(1, nranks):
        target = k * nx / nranks
        cand = legal[legal > cuts[-1] + 3]
        assert len(cand), "block too short for %d slabs" % nranks
        cuts.append(int(cand[np.argmin(np.abs(cand - target))]))
    cuts.append(nx)
    assert all(b - a >= 4 for a, b in zip(cuts[:-1], cuts[1:])), "block too short for %d slabs" % nranks
    i0, i1 = cuts[rank], cuts[rank + 1]
    sc = scene_fn(x_range=(i0, i1), **kw)
    f = sc["fluids"][0]
    ny_nz = len(f["positions"]) // (i1 - i0)
    f["ids"] = (np.arange(len(f["positions"]), dtype=np.int64) + i0 * ny_nz).astype(np.uint32)
    planes = [-2 ** 31] + [int(np.floor((x[k] - amp * 1.001) / float(h))) for k in cuts[1:-1]] + [2 ** 31 - 1]
    sc["slab"] = (planes[rank], planes[rank + 1])
    sc["planes"] = planes
    sc["partitioned"] = True
    return sc


def scene_c5(n=100):
    """2 stacked n^3 blocks (rho0 1000 below, 800 above), IISPH + ArtificialViscosity + Becker2009."""
    r = 0.025
    s = 2.0 * r
    lower = jitter(block_lattice(n, n, n, r), r, 0x5A17A)
    upper = jitter(block_lattice(n, n, n, r, origin=(0.0, n * s, 0.0)), r, 0x5A17A + 1)
    lo = (-r, -r, -r)
    hi = (n * s * 2.0 + r, 2 * n * s + 4 * s + r, n * s + r)
    forces = [artificial_viscosity(1.0, 0.0), becker2009_elasticity(1.0e5, 0.3, True)]
    return dict(name="C5-iisph-2fluid-%d" % (2 * n ** 3), particle_radius=r, smoothing_factor=2.0, dt=1.0 / 1000.0,
                gravity=GRAVITY, solver=IISPH,
                fluids=[dict(positions=lower, density0=1000.0, forces=list(forces)),
                        dict(positions=upper, density0=800.0, forces=list(forces))],
                boundaries=[dict(positions=open_tank(lo, hi, r))])



def populate(world, scene):
    """Feed a scene dict into any world exposing add_fluid/push_force/add_boundary
    (salva_b200.LiquidWorld and oracle.OracleWorld both do).  Returns (fluid handles, boundary handles)."""
    fh, bh = [], []
    for f in scene["fluids"]:
        h = world.add_fluid(f["positions"], density0=f["density0"], velocities=f.get("velocities"),
                            memberships=f.get("memberships", 1), filter=f.get("filter", 0xFFFFFFFF))
        for kind, params in f.get("forces", []):
            world.push_force(h, kind, params)
        fh.append(h)
    for b in scene["boundaries"]:
        bh.append(world.add_boundary(b["positions"], velocities=b.get("velocities"),
                                     memberships=b.get("memberships", 1), filter=b.get("filter", 0xFFFFFFFF),
                                     want_forces=b.get("want_forces", False)))
    return fh, bh
