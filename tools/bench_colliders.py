"""Step time of collider coupling on the device (sph_collider_*, StaticSampling) against the alternatives.

C1: basic3.rs's ground and walls as StaticSampling colliders on a fixed body, against the same particles as plain boundaries.
C2: the 1M-particle dam break with a StaticSampling cuboid (surface samples) that moves through the block every step, three
ways: posed on the device, posed by the host and written with sph_boundary_write, and no collider at all.
The variants of a scene are stepped alternately in one process; the card, its power limit and SM clock are read in the
same run.  Prints one JSON line per scene.

    python tools/bench_colliders.py --steps 50 --warmup 10
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from salva_b200 import BODY_FIXED, DFSPHSolver, LiquidWorld, StaticSampling, scenes  # noqa: E402

F32 = np.float32


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def world_for(sc, boundaries_as):
    w = LiquidWorld(DFSPHSolver(), particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    f = sc["fluids"][0]
    fh = w.add_fluid(f["positions"], density0=f["density0"])
    for kind, params in f["forces"]:
        w.push_force(fh, kind, params)
    colliders = []
    for b in sc["boundaries"]:
        if boundaries_as == "plain":
            w.add_boundary(b["positions"])
        else:  # a fixed collider whose local frame is the particles' centroid
            c0 = b["positions"].mean(axis=0).astype(F32)
            bh = w.add_boundary(np.zeros((0, 3), F32))
            c = w.register_coupling(bh, StaticSampling(b["positions"] - c0))
            w.set_collider_state(c, translation=c0, body=BODY_FIXED)
            colliders.append(c)
    return w


def timed(w, dt, advance=None):
    if advance:
        advance()
    t0 = time.perf_counter()
    w.step(dt)  # ends with a stream synchronise
    wall = (time.perf_counter() - t0) * 1e3
    st = w.stats()
    return st["step_ms"], wall, st["kernel_launches"]


def run(variants, dt, steps, warmup):
    res = {k: [] for k in variants}
    for i in range(warmup + steps):
        for name, (w, adv) in variants.items():
            r = timed(w, dt, adv(i) if adv else None)
            if i >= warmup:
                res[name].append(r)
    out = {}
    for name, rows in res.items():
        a = np.array(rows)
        out[name] = dict(step_ms=float(np.median(a[:, 0])), wall_ms=float(np.median(a[:, 1])), launches=int(a[-1, 2]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--c2", type=int, default=100, help="C2 block edge (100 = 1M particles)")
    a = ap.parse_args()
    gpu = card()

    c1 = scenes.scene_c1()
    print(json.dumps(dict(scene="C1-basic3 tank", gpu=gpu, **run(
        {"plain": (world_for(c1, "plain"), None), "static_colliders": (world_for(c1, "colliders"), None)}, c1["dt"], a.steps, a.warmup))))

    c2 = scenes.scene_c2(a.c2)
    r = c2["particle_radius"]
    box = scenes.cuboid_surface((0.3, 0.3, 0.3), r)
    span = a.c2 * 2 * r

    def pose(i):
        return np.array([0.2 * span + 0.004 * i, 0.5 * span, 0.5 * span], F32)

    dev = world_for(c2, "plain")
    dev_c = dev.register_coupling(dev.add_boundary(np.zeros((0, 3), F32)), StaticSampling(box))
    host = world_for(c2, "plain")
    host_b = host.add_boundary(box + pose(0))
    none = world_for(c2, "plain")

    def dev_adv(i):
        return lambda: dev.set_collider_state(dev_c, translation=pose(i), body=BODY_FIXED)

    def host_adv(i):
        return lambda: host.write_boundary(host_b, box + pose(i))
    print(json.dumps(dict(scene="C2-%d moving cuboid" % a.c2 ** 3, gpu=gpu, **run(
        {"device_collider": (dev, dev_adv), "host_write": (host, host_adv), "no_collider": (none, None)}, c2["dt"], a.steps, a.warmup))))
    print(json.dumps(dict(gpu_after=card())))


if __name__ == "__main__":
    main()
