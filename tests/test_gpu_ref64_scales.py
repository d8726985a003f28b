"""The CUDA engine's gather passes against the float64 per-pass reference (oracle/ref64_stages.py) away from particle radius
0.05 and smoothing factor 2: the scale scenes (ref64_stages.SCALE_SCENES) reach smoothing factors 1, 1.37 and 3 and
h = 0.008, where the gradient gate, the list lengths, the d^2 = h^2 ties and the generic kernels' normalisations differ from
every other scene's (tests/test_ref64_scales.py checks the CPU oracle and the kernel bugs each scene is built for).  Every
check runs in both grid orders and with the generic-kernel library, and prints the worst |err| / bound per pass."""
import json

import numpy as np
import pytest

from oracle import ref64
from oracle import ref64_stages as S
from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, scenes
from salva_b200.liquid_world import Poly6Kernel, SphError, SpikyKernel, ViscosityKernel

pytestmark = pytest.mark.gpu

F = np.float32
K = {1: Poly6Kernel, 2: SpikyKernel, 3: ViscosityKernel}
NAMES = sorted(S.SCALE_SCENES)
# (kernel density, kernel gradient, SALVA_B200_XYSUB): h order, row order, and the generic-kernel library in h order
VARIANTS = {"h_order": (0, 0, "1"), "row_order": (0, 0, "2"), "poly6+spiky": (1, 2, "1"), "viscosity+poly6": (3, 1, "1")}
CHECKS = ("dfsph", "iisph", "tension", "viscosity", "becker", "loops")
# The viscosity kernel vanishes at r = 0 and at r = h, so on sf1_lattice's exact lattice and tank (spacing h) every boundary
# volume sum is zero: the engine refuses the world, as the reference asserts (test_the_viscosity_kernel_refuses_...).
REFUSED = {("sf1_lattice", "viscosity+poly6")}
# A second step after one with pinned loops (the dt change of loop_errors, and DFSPHViscosity after a WCSPH force): the
# first step flings particles of these worlds far beyond the grid (sf1_lattice's 4.6x compressed sub-block, small's edge
# pairs under the viscosity kernel; the CPU oracle too), and the dense grid refuses the next step with SPH_ERR_OOM or a
# particle left alone has zero density.  Their first steps are checked.
ONE_STEP = {("sf1_lattice", v) for v in VARIANTS} | {("small", "viscosity+poly6")}


def _gpu(sc, kd=0, kg=0, solver=DFSPHSolver):
    def make(**kw):
        s = solver(K[kd], K[kg]) if kd else solver()
        for k, v in kw.items():
            setattr(s, k, v)
        return LiquidWorld(s, particle_radius=S.radius(sc), smoothing_factor=S.smoothing(sc))
    return make


def _report(c, **tags):
    print("\nREF64 %s" % json.dumps(dict(tags, worst={k: round(float(v), 5) for k, v in c.worst.items()},
                                         excluded={k: v for k, v in c.excluded.items() if v})))
    assert not c.flagged(), c.worst


@pytest.mark.parametrize("check", CHECKS)
@pytest.mark.parametrize("name,variant", [(n, v) for n in NAMES for v in sorted(VARIANTS) if (n, v) not in REFUSED])
def test_every_pass_meets_its_bound_at_other_scales(name, variant, check, monkeypatch):
    kd, kg, xysub = VARIANTS[variant]
    monkeypatch.setenv("SALVA_B200_XYSUB", xysub)  # read when the world is created
    sc = S.SCALE_SCENES[name]()
    if check == "viscosity":
        sc = S.light(sc)
    solver = IISPHSolver if check == "iisph" else DFSPHSolver
    c = S.Checks(_gpu(sc, kd, kg, solver), sc, kw=kd, kg=kg)
    if check == "dfsph":
        c.stages()
        c.akinci(0.0)
        c.akinci(0.5)
        c.xsph(0.5, 0.3)
        c.artificial(1.0, 0.5, beta=0.3)
        assert c.worst["counts"] == 0
        if name == "sf3":   # lists regrown from 64 past 256
            assert c.nf.max() > 256, c.nf.max()
    elif check == "iisph":
        o = c.iisph_stages()
        if name == "small":   # the isolated pair: two contacts each, and no gradient between them (dii sums it alone)
            iso = list(sc["isolated"])
            assert (c.nf[iso] == 2).all() and (c.nb[iso] == 0).all()
            assert (o["dii"][iso] == 0).all(), o["dii"][iso]
    elif check == "tension":
        c.wcsph(0.5)
        for cf, cb in ((0.5, 0.0), (0.5, 0.3)):
            c.he2014(cf, cb)
    elif check == "viscosity":
        c.viscosity(0.5)
        if (name, variant) not in ONE_STEP:
            c.viscosity(0.5, wcsph=2.0)
    elif check == "becker":
        c.becker(nonlinear=True)
        c.becker(nonlinear=False)
    else:
        c.loop_errors()
        if (name, variant) not in ONE_STEP:
            c.loop_errors((c.dt, 2 * c.dt))
    _report(c, scene=name, variant=variant, check=check)


@pytest.mark.parametrize("name,variant", sorted(REFUSED))
def test_the_viscosity_kernel_refuses_the_sf1_lattice(name, variant, monkeypatch):
    kd, kg, xysub = VARIANTS[variant]
    monkeypatch.setenv("SALVA_B200_XYSUB", xysub)
    sc = S.SCALE_SCENES[name]()
    w = _gpu(sc, kd, kg)()
    S.populate(w, sc)
    with pytest.raises(SphError, match="ZERO_DENSITY"):
        w.step(S.timestep(sc), S.ZERO_G)
    w.close()


def _contacts(sc):
    """One step (0, 0) of a fresh h-order world with a host force that keeps the materialised contacts: positions, and per
    particle the fluid neighbours' indices and gradients (caller order of the context)."""
    seen = {}

    def solve(ctx):
        ff = ctx.fluid_fluid_contacts
        seen.update(pos=ctx.positions.copy(), off=ff.offsets.astype(np.int64).copy(), j=ff.j.astype(np.int64).copy(),
                    grad=ff.gradient.copy())

    w = _gpu(sc)()
    (fh,), _ = S.populate(w, sc)
    w.push_host_force2(fh, solve, boundaries=False)
    w.force_iterations(0, 0)
    w.step(S.timestep(sc), S.ZERO_G)
    bits = np.unique(w.debug(fh, "fluid_list_bits"))
    nf = w.debug(fh, "num_fluid_contacts")
    w.close()
    i = np.repeat(np.arange(len(seen["pos"])), np.diff(seen["off"]))
    return seen, i, bits, nf


def test_the_sf3_lists_grow_past_256_and_stay_narrow(monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "1")
    sc = S.scene_sf3()
    seen, i, bits, nf = _contacts(sc)
    assert nf.max() > 256 and list(bits) == [16], (nf.max(), bits)
    assert np.array_equal(np.sort(nf), np.sort(S.passes_for(sc).nf))


def test_the_sf1_lattice_ties_are_contacts(monkeypatch):
    """Every axis pair of the exact lattice, at d^2 = h^2 in float32, is in the engine's contact lists."""
    monkeypatch.setenv("SALVA_B200_XYSUB", "1")
    sc = S.scene_sf1_lattice()
    seen, i, bits, nf = _contacts(sc)
    P = seen["pos"]
    lat = {tuple(p) for p in scenes.block_lattice(*S.SF1_LATTICE, S.radius(sc)).tolist()}
    on = np.array([tuple(p) in lat for p in P.tolist()])
    assert on.sum() == sc["lattice"]
    h = S.passes_for(sc).h
    h2 = F(F(h) * F(h))
    j = seen["j"]
    tie = (ref64.f32_d2(P[i], P[j]) == h2) & on[i] & on[j]
    assert int(tie.sum()) == S.lattice_ties(S.SF1_LATTICE), (int(tie.sum()), S.lattice_ties(S.SF1_LATTICE))


def test_the_small_isolated_pair_is_a_contact_with_zero_gradient(monkeypatch):
    monkeypatch.setenv("SALVA_B200_XYSUB", "1")
    sc = S.scene_small()
    seen, i, bits, nf = _contacts(sc)
    P = seen["pos"]
    Q = sc["fluids"][0]["positions"]
    a, b = (int(np.nonzero((P == Q[k]).all(1))[0][0]) for k in sc["isolated"])
    for x, y in ((a, b), (b, a)):
        mine = i == x
        assert sorted(seen["j"][mine].tolist()) == sorted([x, y])
        assert (seen["grad"][mine] == 0).all(), seen["grad"][mine]
