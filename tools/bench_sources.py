"""What particle sinks and sources on the device cost and save (sph_fluid_add_sink / sph_fluid_add_source, DESIGN.md section 14).

(a) C2 (the dam break, --c2-n^3 particles) in its tank, with and without a domain sink around the tank that removes nothing,
    in alternating rounds: the per-step overhead of the classification pass and its read-back.
(b) C2 with a 10 000-particle source every 10 steps and a drain sink in a floor corner, against a twin that applies the same
    rule from the host each step (read the positions, delete_particles, append_particles, as faucet3.rs:69-105 does).  The
    two worlds' states must stay bit-identical.

Wall ms per step is a host clock around each round of steps (every step ends in a synchronising read-back).  The card's
name, power limit and SM clock are read in the same run.  Prints one JSON line per part.

    python tools/bench_sources.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from salva_b200 import LiquidWorld, scenes  # noqa: E402

G = (0.0, -9.81, 0.0)
F = np.float32


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def make(n):
    sc = scenes.scene_c2(n)
    w = LiquidWorld(particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh, _ = scenes.populate(w, sc)
    tank = sc["boundaries"][0]["positions"]
    return w, fh[0], sc["dt"], tank


def state(w, f):
    p, v = w.read_fluid(f)
    return p.view(np.uint32).copy(), v.view(np.uint32).copy(), w.read_ids(f), w.debug(f, "velocity_change").view(np.uint32)


def same(a, b):
    return all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def part_a(n, rounds, steps):
    (w0, f0, dt, tank), (w1, f1, _, _) = make(n), make(n)
    lo, hi = tank.min(0) - F(0.5), tank.max(0) + F(0.5)
    w1.add_sink(f1, lo, hi, outside=True)
    ms = {0: [], 1: []}
    launches = {}
    for w in (w0, w1):  # warm-up
        for _ in range(3):
            w.step(dt, G)
    for r in range(rounds):
        for arm in ((0, 1) if r % 2 == 0 else (1, 0)):
            w = (w0, w1)[arm]
            t = time.perf_counter()
            for _ in range(steps):
                w.step(dt, G)
            ms[arm].append((time.perf_counter() - t) * 1e3 / steps)
            launches[arm] = w.stats()["kernel_launches"]
    return dict(part="a", particles=n ** 3, steps_per_round=steps, rounds=rounds, ms_plain=ms[0], ms_sink=ms[1],
                median_plain=float(np.median(ms[0])), median_sink=float(np.median(ms[1])), launches_plain=launches[0],
                launches_sink=launches[1], bit_identical=same(state(w0, f0), state(w1, f1)))


def part_b(n, steps, interval, per):
    (wd, fd, dt, tank), (wh, fh, _, _) = make(n), make(n)
    side = int(round((per // 2) ** 0.5 / 2 ** 0.5)) or 1  # two layers of nx x nz = per / 2 particles, nz = 2 nx
    nx, nz = side, per // 2 // side
    r = F(0.025)
    gx = F(6.0) + np.arange(nx, dtype=F) * F(2) * r
    gz = F(0.025) + np.arange(nz, dtype=F) * F(2) * r
    layers = []
    for y in (F(4.0), F(4.05)):
        p = np.stack(np.meshgrid(gx, np.array([y], F), gz, indexing="ij"), -1).reshape(-1, 3)
        layers.append(p)
    tpl = np.concatenate(layers).astype(F)
    vel = np.zeros_like(tpl)
    vel[:, 1] = -2.0
    lo, hi = np.array([-np.inf, -np.inf, -np.inf], F), np.array([0.5, 0.3, np.inf], F)  # a drain in a floor corner
    wd.add_sink(fd, lo, hi)
    wd.add_source(fd, tpl, vel, interval)
    ms = {"device": [], "host": []}
    removed = emitted = 0
    for k in range(steps):
        t = time.perf_counter()
        wd.step(dt, G)
        ms["device"].append((time.perf_counter() - t) * 1e3)
        e = wd.step_edits(fd)
        removed += e[0]
        emitted += e[1]
        t = time.perf_counter()
        p, _ = wh.read_fluid(fh)
        mask = np.all((lo <= p) & (p < hi), axis=1)
        if mask.any():
            wh.delete_particles(fh, mask)
        if k % interval == 0:
            wh.append_particles(fh, tpl, vel)
        wh.step(dt, G)
        ms["host"].append((time.perf_counter() - t) * 1e3)
    warm = min(interval, steps // 2)
    return dict(part="b", particles=n ** 3, template=len(tpl), interval=interval, steps=steps, removed=removed, emitted=emitted,
                final_particles=wd.num_particles(fd), ms_device_median=float(np.median(ms["device"][warm:])),
                ms_host_median=float(np.median(ms["host"][warm:])), ms_device_mean=float(np.mean(ms["device"][warm:])),
                ms_host_mean=float(np.mean(ms["host"][warm:])), bit_identical=same(state(wd, fd), state(wh, fh)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c2-n", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--b-steps", type=int, default=60)
    ap.add_argument("--interval", type=int, default=10)
    ap.add_argument("--per", type=int, default=10000)
    ap.add_argument("--out", default=None, help="directory for bench_sources.jsonl")
    a = ap.parse_args()
    gpu = card()
    lines = []
    for res in (part_a(a.c2_n, a.rounds, a.steps), part_b(a.c2_n, a.b_steps, a.interval, a.per)):
        res["gpu"] = gpu
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_sources.jsonl"), "w") as fo:
            fo.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
