"""What a device surface extraction costs (sph_world_extract_surface, DESIGN.md section 15).

At C2 (the dam break, --c2-n^3 particles) and C3 (--c3-n^3), each after --settle steps, at spacing r and r / 2: ms per
extraction (device events around the call, median over --rounds after one warm-up), that world's ms per step measured in
the same run (same events around one step), the lattice points, vertices and triangles.  With --profile, a separate run
per configuration under torch.profiler gives the field pass's kernel time; its compulsory bytes (one phi write per lattice
point, each binned particle read once) over that time is reported as a rate.  The card's name, power limit and SM clocks
are read in the same run.  Prints one JSON line per configuration.

With --anisotropic (sph_world_extract_surface_anisotropic, DESIGN.md section 17) it times instead the isotropic and the
anisotropic extraction of the same world, alternating, at C2 spacing r and r / 2 and at C3 spacing r, with normals; with
--profile also the anisotropic extraction's kernel times per pass (ellipsoids, the two binnings, field, normals).

    python tools/bench_surface.py --out DIR [--profile] [--anisotropic]
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
from salva_b200 import LiquidWorld, SurfaceAnisotropy, scenes  # noqa: E402


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


def run(name, sc, settle, rounds, profile, out):
    w = LiquidWorld(particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh, _ = scenes.populate(w, sc)
    dt = sc["dt"]
    for _ in range(settle):
        w.step(dt)
    r = float(sc["particle_radius"])
    n = w.num_particles(fh[0])
    lines = []
    for sp_name, sp in (("r", r), ("r/2", 0.5 * r)):
        w.extract_surface(iso=0.6, spacing=sp)  # warm-up: allocations and module loads
        step_ms, _ = timed(lambda: w.step(dt), rounds)
        ext_ms, all_ms = timed(lambda: w.extract_surface(iso=0.6, spacing=sp), rounds)
        nv, nt = w.extract_surface(iso=0.6, spacing=sp)
        phi, _, _ = w.surface_field()
        rec = dict(scene=name, particles=n, spacing=sp_name, lattice_points=int(phi.size), vertices=nv, triangles=nt,
                   extract_ms=round(ext_ms, 3), extract_ms_rounds=all_ms, step_ms=round(step_ms, 3), card=card())
        if profile:
            from torch.profiler import ProfilerActivity, profile as tprof
            with tprof(activities=[ProfilerActivity.CUDA]) as prof:
                w.extract_surface(iso=0.6, spacing=sp)
                torch.cuda.synchronize()
            us = sum(e.device_time_total for e in prof.key_averages() if "k_surf_field" in e.key)
            bytes_ = 4 * phi.size + 16 * n
            rec.update(field_kernel_ms=round(us / 1000.0, 3), field_compulsory_GBps=round(bytes_ / (us * 1e-6) / 1e9, 1) if us else None)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    w.close()
    with open(os.path.join(out, "bench_surface_%s.json" % name), "w") as f:
        json.dump(lines, f, indent=1)


PASSES = {"ellipsoids": ("k_surf_ellipsoids",), "binning_and_scans": ("k_surf_hist", "k_cell_scatter", "k_surf_cell_sort", "k_gather", "k_scan"),
          "field": ("k_surf_field_aniso",), "normals": ("k_surf_normals_aniso",), "polygonise": ("k_surf_count", "k_surf_emit")}


def run_aniso(name, sc, spacings, settle, rounds, profile, out):
    """Isotropic and anisotropic extraction of one settled world, alternating round by round."""
    w = LiquidWorld(particle_radius=sc["particle_radius"], smoothing_factor=sc["smoothing_factor"])
    fh, _ = scenes.populate(w, sc)
    for _ in range(settle):
        w.step(sc["dt"])
    r = float(sc["particle_radius"])
    an = SurfaceAnisotropy()
    lines = []
    for sp_name in spacings:
        sp = r if sp_name == "r" else 0.5 * r
        iso = lambda: w.extract_surface(iso=0.6, spacing=sp)  # noqa: E731
        ani = lambda: w.extract_surface(iso=0.6, spacing=sp, anisotropy=an)  # noqa: E731
        iso()
        ani()  # warm-up: allocations and module loads
        t_iso, t_ani = [], []
        for _ in range(rounds):
            t_iso.append(timed(iso, 1)[0])
            t_ani.append(timed(ani, 1)[0])
        nv, nt = ani()
        rec = dict(scene=name, particles=w.num_particles(fh[0]), spacing=sp_name, vertices_aniso=nv, triangles_aniso=nt,
                   iso_ms=round(float(np.median(t_iso)), 3), aniso_ms=round(float(np.median(t_ani)), 3),
                   iso_ms_rounds=[round(x, 3) for x in t_iso], aniso_ms_rounds=[round(x, 3) for x in t_ani], card=card())
        if profile:
            from torch.profiler import ProfilerActivity, profile as tprof
            with tprof(activities=[ProfilerActivity.CUDA]) as prof:
                ani()
                torch.cuda.synchronize()
            ev = prof.key_averages()
            rec["aniso_pass_ms"] = {k: round(sum(e.device_time_total for e in ev if any(n in e.key for n in names)) / 1000.0, 3)
                                    for k, names in PASSES.items()}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    w.close()
    with open(os.path.join(out, "bench_surface_aniso_%s.json" % name), "w") as f:
        json.dump(lines, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for bench_surface_*.json (default: a temporary one)")
    ap.add_argument("--c2-n", type=int, default=100)
    ap.add_argument("--c3-n", type=int, default=216)
    ap.add_argument("--settle", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--anisotropic", action="store_true", help="isotropic against anisotropic extraction, alternating")
    a = ap.parse_args()
    if a.out is None:
        import tempfile
        a.out = tempfile.mkdtemp(prefix="bench_surface_")
    os.makedirs(a.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("bench_surface needs a CUDA device")
    if a.anisotropic:
        run_aniso("C2", scenes.scene_c2(a.c2_n), ("r", "r/2"), a.settle, a.rounds, a.profile, a.out)
        run_aniso("C3", scenes.scene_c3(a.c3_n), ("r",), a.settle, a.rounds, a.profile, a.out)
        return
    run("C2", scenes.scene_c2(a.c2_n), a.settle, a.rounds, a.profile, a.out)
    run("C3", scenes.scene_c3(a.c3_n), a.settle, a.rounds, a.profile, a.out)


if __name__ == "__main__":
    main()
