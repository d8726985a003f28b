"""Step time of DynamicContactSampling on the device (SPH_SAMPLING_CONTACT) against the same rule run as a host
CouplingManager (salva_b200.contact_sampling.ContactSamplingHook through step_with_coupling) and against no collider.

C2: the 1M-particle dam break (DFSPH + XSPH) with a 0.6 m cuboid on a dynamic body that moves through the block every step.
Droplet: examples/contact_sampling3.cpp's scene (surface_tension3.rs, a 7^3 droplet on a fixed cuboid ground).
C2 again with a moving cylinder and a moving cone, after the two scenes above, whose output does not change.
The variants of a scene are stepped alternately in one process; the card, its power limit and SM clock are read in the
same run.  Prints one JSON line per scene: median step ms (CUDA events), median wall ms and kernels per step.

    python tools/bench_contact_sampling.py --steps 100 --warmup 10
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from salva_b200 import BODY_DYNAMIC, BODY_FIXED, DFSPHSolver, DynamicContactSampling, LiquidWorld, scenes  # noqa: E402
from salva_b200.contact_sampling import ContactSamplingHook  # noqa: E402
from salva_b200.liquid_world import Cone, Cuboid, Cylinder  # noqa: E402

F32 = np.float32


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def run(variants, dt, gravity, steps, warmup):
    """variants: name -> (world, advance(i) -> step function)"""
    res = {k: [] for k in variants}
    for i in range(warmup + steps):
        for name, (w, adv) in variants.items():
            step = adv(i)
            t0 = time.perf_counter()
            step()  # every step ends with a stream synchronise
            wall = (time.perf_counter() - t0) * 1e3
            st = w.stats()
            if i >= warmup:
                res[name].append((st["step_ms"], wall, st["kernel_launches"]))
    out = {}
    for name, rows in res.items():
        a = np.array(rows)
        out[name] = dict(step_ms=float(np.median(a[:, 0])), wall_ms=float(np.median(a[:, 1])), launches=int(np.median(a[:, 2])))
    return out


class CountingHook(ContactSamplingHook):
    calls = 0

    def update_boundaries(self, *a):
        super().update_boundaries(*a)
        self.calls += 1


def scene_variants(make, shape, state, dt, gravity):
    """The three variants of one scene: make() -> (world, fluid handles); state(i) -> collider state dict."""
    dev, _ = make()
    dev_c = dev.register_coupling(dev.add_boundary(np.zeros((0, 3), F32)), DynamicContactSampling(shape))
    host, hf = make()
    host_b = host.add_boundary(np.zeros((0, 3), F32), want_forces=state(0)["body"] == BODY_DYNAMIC)
    hook = CountingHook(hf, [(host_b, dict(kind=shape.kind, params=shape.params, **state(0)))])
    none, _ = make()

    def dev_adv(i):
        dev.set_collider_state(dev_c, **state(i))
        return lambda: dev.step(dt, gravity)

    def host_adv(i):
        hook.entries = [(host_b, dict(kind=shape.kind, params=shape.params, **state(i)))]

        def step():
            before = hook.calls
            host.step_with_coupling(dt, gravity, hook)
            assert hook.calls == before + 1, "the host hook failed"  # exceptions inside the callback do not propagate
        return step

    return {"device": (dev, dev_adv), "host_hook": (host, host_adv), "no_collider": (none, lambda i: (lambda: none.step(dt, gravity)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--c2", type=int, default=100, help="C2 block edge (100 = 1M particles)")
    a = ap.parse_args()
    gpu = card()

    c2 = scenes.scene_c2(a.c2)
    r = c2["particle_radius"]
    span = a.c2 * 2 * r

    def make_c2():
        w = LiquidWorld(DFSPHSolver(), particle_radius=r, smoothing_factor=c2["smoothing_factor"])
        f = c2["fluids"][0]
        fh = w.add_fluid(f["positions"], density0=f["density0"])
        for kind, params in f["forces"]:
            w.push_force(fh, kind, params)
        for b in c2["boundaries"]:
            w.add_boundary(b["positions"])
        return w, [fh]

    def c2_state(i):
        t = np.array([0.2 * span + 0.004 * i, 0.5 * span, 0.5 * span], F32)
        return dict(translation=t, rotation=np.eye(3, dtype=F32), body=BODY_DYNAMIC, linvel=np.array([0.004 / c2["dt"], 0.0, 0.0], F32), world_com=t)
    print(json.dumps(dict(scene="C2-%d moving 0.6 m cuboid" % a.c2 ** 3, gpu=gpu, **run(
        scene_variants(make_c2, Cuboid((0.3, 0.3, 0.3)), c2_state, c2["dt"], c2["gravity"]), c2["dt"], c2["gravity"], a.steps, a.warmup))),
        flush=True)

    pr = 0.005

    def make_drop():
        w = LiquidWorld(DFSPHSolver(), particle_radius=pr, smoothing_factor=2.0)
        n, half = 7, 7 * pr
        g = (np.arange(n) * 2 * pr + pr - half).astype(F32)
        pts = np.stack(np.meshgrid(g, g + F32(0.08), g, indexing="ij"), axis=-1).reshape(-1, 3).astype(F32)
        fh = w.add_fluid(pts, density0=1000.0)
        w.push_force(fh, *scenes.akinci2013_surface_tension(1.0, 0.0))
        w.push_force(fh, *scenes.artificial_viscosity(0.01, 0.01))
        return w, [fh]

    def drop_state(i):
        return dict(translation=np.zeros(3, F32), rotation=np.eye(3, dtype=F32), body=BODY_FIXED)
    print(json.dumps(dict(scene="contact_sampling3 droplet", gpu=gpu, **run(
        scene_variants(make_drop, Cuboid((0.15, 0.02, 0.15)), drop_state, 1.0 / 200.0, (0.0, -0.981, 0.0)), 1.0 / 200.0, (0.0, -0.981, 0.0),
        a.steps, a.warmup))), flush=True)
    for shape, label in ((Cylinder(0.3, 0.3), "cylinder"), (Cone(0.3, 0.3), "cone")):  # k_contact_sample<false, true>
        print(json.dumps(dict(scene="C2-%d moving 0.6 m %s" % (a.c2 ** 3, label), gpu=gpu, **run(
            scene_variants(make_c2, shape, c2_state, c2["dt"], c2["gravity"]), c2["dt"], c2["gravity"], a.steps, a.warmup))), flush=True)
    print(json.dumps(dict(gpu_after=card())))


if __name__ == "__main__":
    main()
