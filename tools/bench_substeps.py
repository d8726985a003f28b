"""Cost and effect of CFL-bounded substeps (sph_world_set_substepping, DESIGN.md section 12).

default   bench.py --dump-outputs for C2 and C3 with this tree's library and with --parent-lib (a build of the parent
          commit, given as SALVA_B200_LIB), alternated: whether the default (substepping off) path computes the same bits,
          and its ms/step on both.
c2        C2 given a velocity field that forces 3-4 substeps at T = 1/60: ms per substepped step against the same dt_k
          stepped by hand, and k_cfl_max's time (torch.profiler, CUDA activities, a separate run) against its 32 B per
          particle of compulsory traffic.
dense     DESIGN.md section 7's 10 % over-dense C2 block stepped at 1/60 with and without substepping: the largest speed and
          grid_dims over time, reported only.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line per part.

    python tools/bench_substeps.py --parent-lib /path/to/parent/libsalva_b200.so --out DIR
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from salva_b200 import DFSPHSolver, LiquidWorld, SphError, scenes  # noqa: E402

F32 = np.float32
T = 1.0 / 60.0
G = (0.0, -9.81, 0.0)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def default_path(cfg, parent_lib, steps, warmup, reps, grid_order):
    """bench.py of this tree and of the parent library, alternated `reps` times; the last dumps compared bitwise.  The grid
    order is pinned: bench.py's `auto` picks the faster one per run, and the two orders sum in different orders."""
    ms = {"this": [], "parent": []}
    dumps = {}
    tmp = tempfile.mkdtemp(prefix="bench_substeps_dumps_")
    for rep in range(reps):
        for arm in ("parent", "this"):
            env = dict(os.environ)
            env.pop("SALVA_B200_LIB", None)
            if arm == "parent":
                env["SALVA_B200_LIB"] = parent_lib
            d = os.path.join(tmp, "%s_%s" % (cfg, arm))
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--config", cfg, "--steps", str(steps), "--warmup",
                   str(warmup), "--no-cpu", "--no-parity", "--no-settled", "--grid-order", grid_order, "--dump-outputs", d]
            r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
            lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
            if r.returncode != 0 or not lines:
                raise RuntimeError("bench.py (%s, %s) failed: %s" % (cfg, arm, r.stderr[-2000:]))
            line = json.loads(lines[-1])
            ms[arm].append(line.get("ms_per_step", line.get("value")))
            dumps[arm] = d
    files = sorted(f for f in os.listdir(dumps["this"]) if f.endswith(".npy"))
    same = {f: bool(np.array_equal(np.load(os.path.join(dumps["this"], f)).view(np.uint8),
                                   np.load(os.path.join(dumps["parent"], f)).view(np.uint8))) for f in files}
    shutil.rmtree(tmp, ignore_errors=True)
    return dict(part="default", config=cfg, grid_order=grid_order, ms_per_step=ms, npy_files=len(files), bit_identical=all(same.values()) and bool(files),
                differing=[f for f, s in same.items() if not s])


def c2_world(n, speed, substep, cfl=0.4):
    sc = scenes.scene_c2(n)
    f = sc["fluids"][0]
    pos = f["positions"]
    # a shear field: the top layers move along x at up to `speed`, the bottom ones against it
    y = (pos[:, 1] - pos[:, 1].min()) / max(float(np.ptp(pos[:, 1])), 1e-6)
    vel = np.zeros_like(pos)
    vel[:, 0] = speed * (2.0 * y - 1.0)
    w = LiquidWorld(DFSPHSolver(), particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh = w.add_fluid(pos, density0=f["density0"], velocities=vel.astype(F32))
    for kind, params in f["forces"]:
        w.push_force(fh, kind, params)
    for b in sc["boundaries"]:
        w.add_boundary(b["positions"])
    if substep:
        w.set_substepping(cfl, 1, 10)
    return w, fh, len(pos)


def c2_substepped(n, speed, steps, warmup):
    """A substepped against B stepping A's dt_k by hand (the same work, bit-identical states), alternated step by step."""
    a, _, npart = c2_world(n, speed, True)
    b, _, _ = c2_world(n, speed, False)
    ta, tb, counts, cfl_launch = [], [], [], []
    for k in range(warmup + steps):
        t0 = time.perf_counter()
        a.step(T, G)   # ends with a host synchronisation
        t1 = time.perf_counter()
        dts = a.substeps()
        t2 = time.perf_counter()
        for dt in dts:
            b.step(float(dt), G)
        t3 = time.perf_counter()
        if k >= warmup:
            ta.append((t1 - t0) * 1e3)
            tb.append((t3 - t2) * 1e3)
            counts.append(len(dts))
    # k_cfl_max's device time, in a profiled run of its own
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            a.step(T, G)
            cfl_launch.append(len(a.substeps()))
    kern = [e for e in prof.events() if e.name.startswith("k_cfl_max") or "k_cfl_max" in e.name]
    us = [e.device_time if hasattr(e, "device_time") else e.cuda_time for e in kern]
    mean_us = float(np.mean(us)) if us else None
    bytes_ = 32.0 * npart
    return dict(part="c2", particles=npart, shear_speed=speed, substeps_per_step=counts,
                ms_substepped=dict(median=float(np.median(ta)), min=float(np.min(ta))),
                ms_manual=dict(median=float(np.median(tb)), min=float(np.min(tb))),
                k_cfl_max=dict(launches=len(us), expected=int(sum(cfl_launch)), mean_us=mean_us,
                               compulsory_bytes=bytes_, gb_per_s=(bytes_ / (mean_us * 1e-6) / 1e9) if mean_us else None))


def dense(n, steps):
    out = {}
    for arm in ("off", "on"):
        sc = scenes._dam_break(n, n, n, 0.025, T, [scenes.xsph_viscosity(0.5, 0.0)], name="dense", compress=0.90)
        w = LiquidWorld(DFSPHSolver(), particle_radius=0.025, smoothing_factor=2.0)
        (fh,), _ = scenes.populate(w, sc)
        if arm == "on":
            w.set_substepping(0.4, 1, 10)
        rows = []
        for k in range(steps):
            try:
                w.step(T, G)
            except SphError as e:
                rows.append(dict(step=k, error=str(e)[:200]))
                break
            _, v = w.read_fluid(fh)
            s = w.stats()
            rows.append(dict(step=k, max_speed=float(np.sqrt((v.astype(np.float64) ** 2).sum(1)).max()), grid_dims=s["grid_dims"],
                             n_substeps=s["n_substeps"], step_ms=s["step_ms"]))
        out[arm] = rows
        w.close()
    return dict(part="dense", lattice=n, dt=T, runs=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="default,c2,dense")
    ap.add_argument("--parent-lib", default=None, help="libsalva_b200.so built from the parent commit (part 'default')")
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--grid-orders", default="h,rows", help="bench.py --grid-order values of part 'default'")
    ap.add_argument("--out", default=None, help="directory for bench_substeps.jsonl (default: a temporary one)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--n", type=int, default=100, help="C2 lattice edge")
    ap.add_argument("--speed", type=float, default=4.0)
    ap.add_argument("--dense-steps", type=int, default=30)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="bench_substeps_")
    os.makedirs(out, exist_ok=True)
    lines = [dict(part="card", card=card())]
    parts = args.parts.split(",")
    if "default" in parts:
        if not args.parent_lib:
            raise SystemExit("part 'default' needs --parent-lib")
        for cfg in args.configs.split(","):
            for order in args.grid_orders.split(","):
                lines.append(default_path(cfg, os.path.abspath(args.parent_lib), args.steps, args.warmup, args.reps, order))
                print(json.dumps(lines[-1]), flush=True)
    if "c2" in parts:
        lines.append(c2_substepped(args.n, args.speed, args.steps, args.warmup))
        print(json.dumps(lines[-1]), flush=True)
    if "dense" in parts:
        lines.append(dense(args.n, args.dense_steps))
        print(json.dumps(lines[-1]), flush=True)
    print(json.dumps(lines[0]), flush=True)
    with open(os.path.join(out, "bench_substeps.jsonl"), "w") as fh:
        for l in lines:
            fh.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
