"""What vorticity confinement costs a step (SPH_FORCE_VORTICITY_CONFINEMENT, DESIGN.md section 18).

Twin worlds of one scene, one without and one with the force pushed after the scene's own forces, settled for --settle steps
each; then --rounds rounds that step each twin --steps times, alternating the twins, so that the load of the shared host and
the card's clocks fall on both alike.  Per twin: the median over rounds of ms per step (device events around the steps) and
of step_ms and nonpressure_ms from sph_step_stats (the last step of the round).  The card's name, power limit and SM clocks
are read in the same run.  Prints one JSON line per scene; repeat the command to see the spread between runs.

    python tools/bench_vorticity.py [--scenes c2 c3] [--eps 0.05]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from salva_b200 import LiquidWorld, scenes  # noqa: E402

SCENES = dict(c2=scenes.scene_c2, c3=scenes.scene_c3)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def world(sc, eps):
    w = LiquidWorld(particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh, _ = scenes.populate(w, sc)
    if eps:
        w.push_force(fh[0], *scenes.vorticity_confinement(eps))
    return w


def measure(name, eps, settle, rounds, steps):
    sc = SCENES[name]()
    dt = sc["dt"]
    twins = dict(without=world(sc, 0.0), with_vc=world(sc, eps))
    for w in twins.values():
        for _ in range(settle):
            w.step(dt)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rec = {k: dict(ms=[], step_ms=[], nonpressure_ms=[]) for k in twins}
    for _ in range(rounds):
        for k, w in twins.items():
            a.record()
            for _ in range(steps):
                w.step(dt)
            b.record()
            b.synchronize()
            st = w.stats()
            rec[k]["ms"].append(a.elapsed_time(b) / steps)
            rec[k]["step_ms"].append(st["step_ms"])
            rec[k]["nonpressure_ms"].append(st["nonpressure_ms"])
    n = int(sum(f["positions"].shape[0] for f in sc["fluids"]))
    out = dict(scene=sc.get("name", name), particles=n, eps=eps, rounds=rounds, steps_per_round=steps, card=card())
    for k, r in rec.items():
        out[k] = {m: round(float(np.median(v)), 4) for m, v in r.items()}
        out[k]["ms_rounds"] = [round(x, 4) for x in r["ms"]]
    out["vc_ms_per_step"] = round(out["with_vc"]["ms"] - out["without"]["ms"], 4)
    out["vc_nonpressure_ms"] = round(out["with_vc"]["nonpressure_ms"] - out["without"]["nonpressure_ms"], 4)
    for w in twins.values():
        w.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", nargs="+", default=["c2", "c3"], choices=sorted(SCENES))
    ap.add_argument("--eps", type=float, default=0.05)
    ap.add_argument("--settle", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_vorticity: no CUDA device; nothing is measured without one")
    for name in a.scenes:
        print(json.dumps(measure(name, a.eps, a.settle, a.rounds, a.steps)), flush=True)


if __name__ == "__main__":
    main()
