"""What a device diffuse-particle update costs (sph_world_update_diffuse, DESIGN.md section 16).

C2 (the dam break, --c2-n^3 particles) with a shear field written over its velocities, which generates whitewater.  For each
diffuse capacity in --populations the set is filled by updates (at most --fill of them), then: ms per update (device events
around the call, median over --rounds), that world's ms per step measured in the same run, and the set's size.  With
--profile, a separate run per population under torch.profiler gives each pass's kernel time and its compulsory bytes (every
array a pass must read or write once) over that time as a rate.  The card's name, power limit and SM clocks are read in
the same run.  Prints one JSON line per population.

    python tools/bench_diffuse.py --out DIR [--profile]
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

# thresholds for r = 0.025 (C2): E_k = 0.5 V rho0 |v|^2 with V = 1.25e-5 m^3
DESC = dict(ta_min=0.5, ta_max=4.0, wc_min=0.2, wc_max=2.0, k_min=0.005, k_max=0.1, k_ta=2000.0, k_wc=2000.0, lifetime=4.0)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def timed(fn, rounds):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), [round(x, 3) for x in ms]


def compulsory_bytes(n_fluid, n_diffuse, emitted):
    """Bytes each pass must move at least once: 16 B per float4, 4 per u32 / f32, 8 per u64; the published set is 29 B a
    particle (xyz, xyz, kind, life), the advected one 32 (two float4)."""
    return {
        "k_diffuse_normals": n_fluid * (16 + 16),                                   # binned x; normal out
        "k_diffuse_potentials": n_fluid * (16 * 3 + 4 + 8 + 8 + 12 + 16),           # x, v, n; perm, key; count, normal, 4 values out
        "k_diffuse_emit": n_fluid * 8 + emitted * 32,                               # offsets; emitted rows
        "k_diffuse_advect": n_fluid * 32 + n_diffuse * (29 + 32 + 4),               # binned x, v; set in, advected set out, keep
        "k_diffuse_compact": n_diffuse * (32 + 4 + 29),
    }


def run(sc, populations, fill, rounds, settle, profile, out):
    w = LiquidWorld(particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh, _ = scenes.populate(w, sc)
    f = fh[0]
    p, _ = w.read_fluid(f)
    c = p.mean(axis=0)
    w.write_fluid(f, velocities=np.stack([4.0 * (p[:, 1] - c[1]), np.zeros(len(p)), 2.0 * (p[:, 0] - c[0])], 1).astype(np.float32))
    dt = sc["dt"]
    for _ in range(settle):
        w.step(dt)
    n = w.num_particles(f)
    lines = []
    for cap in populations:
        w.clear_diffuse()
        for _ in range(fill):
            w.update_diffuse(dt, capacity=cap, **DESC)
            if len(w.diffuse_particles()[3]) >= 0.9 * cap:
                break
        step_ms, _ = timed(lambda: w.step(dt), rounds)
        upd_ms, all_ms = timed(lambda: w.update_diffuse(dt, capacity=cap, **DESC), rounds)
        st = w.update_diffuse(dt, capacity=cap, **DESC)
        nd = len(w.diffuse_particles()[3])
        rec = dict(scene="C2-shear", particles=n, capacity=cap, diffuse=nd, stats=st, update_ms=round(upd_ms, 3), update_ms_rounds=all_ms,
                   step_ms=round(step_ms, 3), card=card())
        if profile:
            from torch.profiler import ProfilerActivity, profile as tprof
            with tprof(activities=[ProfilerActivity.CUDA]) as prof:
                st = w.update_diffuse(dt, capacity=cap, **DESC)
                torch.cuda.synchronize()
            by = compulsory_bytes(n, nd, st["emitted"])
            passes = {}
            for e in prof.key_averages():
                name = next((k for k in list(by) + ["k_surf_collect", "k_surf_hist", "k_cell_scatter", "k_surf_cell_sort", "k_gather",
                                                    "k_surf_aabb", "k_scanK"] if k in e.key), None)
                if name:
                    us = passes.get(name, (0.0,))[0] + e.device_time_total
                    passes[name] = (us,)
            rec["passes"] = {k: dict(ms=round(us / 1000.0, 4), compulsory_GBps=round(by[k] / (us * 1e-6) / 1e9, 1) if k in by and us else None)
                             for k, (us,) in passes.items()}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    w.close()
    with open(os.path.join(out, "bench_diffuse.json"), "w") as fp:
        json.dump(lines, fp, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for bench_diffuse.json (default: a temporary one)")
    ap.add_argument("--c2-n", type=int, default=100)
    ap.add_argument("--populations", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--fill", type=int, default=60)
    ap.add_argument("--settle", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if a.out is None:
        import tempfile
        a.out = tempfile.mkdtemp(prefix="bench_diffuse_")
    os.makedirs(a.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("bench_diffuse needs a CUDA device")
    run(scenes.scene_c2(a.c2_n), a.populations, a.fill, a.rounds, a.settle, a.profile, a.out)


if __name__ == "__main__":
    main()
