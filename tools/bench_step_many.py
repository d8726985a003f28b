"""What running steps 2..K of a call as one CUDA graph saves (sph_world_step_many, DESIGN.md section 13).

For C1 (basic3, 3 375 particles) and C2 (the dam break, --c2-n^3 particles), two twin worlds advance in rounds: one by K calls
of step, the other by one step_many(K), alternating which arm goes first, with K in --ks.  Each arm is warmed up (module load,
graph capture) before the timed rounds.  Per arm and K it reports device ms per step (CUDA events around the round), wall ms
per step (host clock around the round, which ends in a synchronising read), host kernel launches per step, the wall time of
the first (untimed) round of each arm, which for step_many includes capturing and instantiating its graph, and whether the
two worlds' positions and velocities stayed bit-identical.  The card's name, power limit and SM clock are read in the same
run.  Prints one JSON line per (config, K).

    python tools/bench_step_many.py --out DIR
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


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def make(cfg, c2_n):
    if cfg == "c1":
        sc, r, dt = scenes.scene_c1(), 0.05, 1.0 / 200.0
        w = LiquidWorld(particle_radius=r, smoothing_factor=2.0)
        fh, _ = scenes.populate(w, sc)
        return w, fh[0], dt
    sc = scenes.scene_c2(c2_n)
    w = LiquidWorld(particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh, _ = scenes.populate(w, sc)
    return w, fh[0], sc.get("dt", 1.0 / 1000.0)


def run_round(w, fh, dt, K, many):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches = 0
    t0 = time.perf_counter()
    e0.record()
    if many:
        assert w.step_many(dt, K) == K
        launches += w.stats()["kernel_launches"]
        on = sum(r["on_device"] for r in w.step_records())
    else:
        for _ in range(K):
            w.step(dt, G)
            launches += w.stats()["kernel_launches"]
        on = 0
    e1.record()
    p, _ = w.read_fluid(fh)  # synchronising read
    wall = time.perf_counter() - t0
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), wall * 1e3, launches, on


def bench(cfg, K, rounds, warmup, c2_n):
    a, fa, dt = make(cfg, c2_n)
    b, fb, _ = make(cfg, c2_n)
    first = {}
    for i in range(warmup):
        sa = run_round(a, fa, dt, K, False)
        sb = run_round(b, fb, dt, K, True)
        if i == 0:  # step_many's first call includes the capture and instantiation of its graph
            first = dict(step=sa[1], step_many=sb[1])
    acc = {False: [0.0, 0.0, 0, 0], True: [0.0, 0.0, 0, 0]}
    for r in range(rounds):
        for many in ((False, True) if r % 2 == 0 else (True, False)):
            w, fh = (b, fb) if many else (a, fa)
            dev, wall, launches, on = run_round(w, fh, dt, K, many)
            s = acc[many]
            s[0] += dev
            s[1] += wall
            s[2] += launches
            s[3] += on
    same = all(np.array_equal(x, y) for x, y in zip(a.read_fluid(fa), b.read_fluid(fb)))
    n = rounds * K
    arm = lambda s: dict(device_ms_per_step=s[0] / n, wall_ms_per_step=s[1] / n, launches_per_step=s[2] / n)
    return dict(config=cfg, K=K, rounds=rounds, step=arm(acc[False]), step_many=dict(arm(acc[True]), on_device_steps=acc[True][3],
                steps=n), first_round_wall_ms=first, bit_identical=same, card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c1,c2")
    ap.add_argument("--ks", default="8,64")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--c2-n", type=int, default=100)
    ap.add_argument("--out", default=None, help="directory for bench_step_many.jsonl")
    a = ap.parse_args()
    lines = []
    for cfg in a.configs.split(","):
        for K in [int(k) for k in a.ks.split(",")]:
            res = bench(cfg, K, a.rounds, a.warmup, a.c2_n)
            print(json.dumps(res), flush=True)
            lines.append(res)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_step_many.jsonl"), "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
