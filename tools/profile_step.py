"""Per-kernel device time of a few warm steps of a bench workload, grouped by phase, with the bytes the streaming kernels move.

    python tools/profile_step.py [--config c3] [--steps 3] [--warmup 3] [--out DIR]

Runs the workload bench.py builds (C3 by default: 10 077 696 particles, DFSPH + Akinci2013) under torch.profiler with CUDA
activities and prints, per kernel: launches per step, device ms per step, bytes per step from the byte model below, and the
achieved GB/s.  The card name and power limit (read-only nvidia-smi query) are printed with the table: they are part of every
number in it.  The trace goes under --out (default: a temporary directory).

BYTES is the per-particle traffic of one launch of each streaming kernel as the code stores and loads it, for a single
uniform-mass fluid (C2, C3): reads + writes, with sector-wide loads of a float4 counted whole.  The uniform-mass Jacobi gather
passes (GATHER_OWN) count their own records plus the fluid lists they stream once (list_bytes: the counts and every stored
group, in the width the last search chose, sph_lists.cuh); the neighbour records they gather are served by L1/L2 and are not
counted.  Scans and the other passes have no entry: their traffic depends on the grid, so only their time is printed.
"""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BYTES = {
    "k_cell_hist": 16 + 8,                    # pos; cid, rank
    "k_cell_hist_xy": 16 + 8,
    "k_cell_scatter": 12 + 4 + 4 + 8,         # cid, rank, start[c]; gid; perm, key (scattered)
    "k_cell_sort": 12,                        # key, perm (entries that move are written back as well)
    "k_gather_vstar": 4 + 48 + 8 + 48 + 8 + 16 + 8,  # perm, pos/vel/vc, orig/gid; pos/vel/vc, orig/gid, pvx4, vyz2
    "k_fold_integrate": 16 + 16 + 8 + 16 + 48 + 16 + 8,  # vel, pvx4, vyz2, xs; vel/acc/vc, pvx4, vyz2
    "k_fold_velocities": 16 + 16 + 8 + 16 + 48,          # vel, pvx4, vyz2, xs; vel/acc/vc
    "k_integrate_acc": 48 + 16 + 8 + 4,                  # acc, vc, vel; vc, vyz2, pvx4.w
    "k_update_positions": 16 + 16 + 8 + 16,              # pos, pvx4, vyz2; pos
}

# own records of the uniform-mass Jacobi passes per particle and launch (reads; writes)
GATHER_OWN = {
    "k_vel_update_u": 16 + 16 + 16 + 16 + 16 + 8,         # pk4, vel, vc; vc, pvx4, vyz2
    "k_vel_divergence_u": 16 + 8 + 4 + 4 + 4 + 16,        # pvx4, vyz2, alpha, dens (predicted); out, pk4
    "k_vel_divergence_xsph_u": 16 + 8 + 4 + 16 + 4 + 16 + 16,  # pvx4, vyz2, alpha, nr4; divv, pk4, xs
}


def list_bytes(counts, bits):
    """Bytes one pass streams from the fluid lists: the two counts per particle, and per stored group of four entries 16 B
    (32-bit entries) or 8 B plus 12 B of window bases per particle (16-bit entries)."""
    groups = int(((counts + 3) // 4).sum())
    return 8 * len(counts) + (16 * groups if bits == 32 else 8 * groups + 12 * len(counts))


PHASES = [
    ("grid", ("k_bounds", "k_cell_hist", "k_cell_hist_xy", "k_scan_block", "k_scan_add", "k_scanK_block", "k_scanK_add",
              "k_cell_scatter", "k_cell_sort", "k_gather_vstar", "k_gather")),
    ("neighbours + density", ("k_neighbors", "k_neighbors_xy", "k_lists_check")),
    ("divergence update", ("k_vel_update_u@div", "k_vel_update@div")),
    ("divergence evaluation", ("k_vel_divergence_u<false>", "k_vel_divergence_xsph_u")),
    ("predicted density", ("k_vel_divergence_u<true>",)),
    ("pressure update", ("k_vel_update_u@press", "k_vel_update@press")),
    ("tail", ("k_fold_integrate", "k_fold_velocities", "k_integrate_acc", "k_cfl_max", "k_update_positions", "k_bounds_init",
              "k_reduce_partials", "k_loop_decide", "k_fold_arm", "k_graph_arm", "k_step_end")),
]


def gpu_info():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as e:  # nvidia-smi missing: the numbers still print, without their card
        return {"error": str(e)[:100]}


def kernel_key(name):
    """Base kernel name, with the template arguments that tell the Jacobi passes apart kept (k_vel_update_u<BFORCE, PRESSURE, ..>)."""
    m = re.search(r"(k_\w+)(<[^()]*>)?", name)
    if not m:
        return name[:60]
    base, targs = m.group(1), m.group(2) or ""
    if base in ("k_vel_update_u", "k_vel_update"):
        a = [t.strip() for t in targs.strip("<>").split(",")]
        pressure = a[1] if base == "k_vel_update_u" else (a[2] if len(a) > 2 else "false")
        return base + ("@press" if pressure == "true" else "@div")
    if base == "k_vel_divergence_u":
        return base + targs
    return base


def phase_of(key):
    for ph, names in PHASES:
        for n in names:
            if key == n or key.startswith(n):
                return ph
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3", choices=["c2", "c3", "c5"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--grid-order", default="h", choices=["h", "rows"])
    ap.add_argument("--out", default=None, help="directory for the trace (default: a temporary one)")
    ap.add_argument("--json", default=None, help="also write the table as JSON to this file")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a CUDA device")
    os.environ["SALVA_B200_XYSUB"] = "2" if args.grid_order == "rows" else "1"
    import bench
    from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, scenes

    sc = bench.build_scene(args.config)
    world = LiquidWorld(DFSPHSolver() if sc["solver"] == 0 else IISPHSolver(), particle_radius=sc["particle_radius"],
                        smoothing_factor=sc["smoothing_factor"], device=0, deterministic=True)
    fh, _ = scenes.populate(world, sc)
    n = sum(world.num_particles(f) for f in fh)
    for _ in range(max(args.warmup, 1)):
        world.step(sc["dt"], sc["gravity"])
    torch.cuda.synchronize()
    step_ms = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            world.step(sc["dt"], sc["gravity"])
            step_ms.append(world.stats()["step_ms"])
        torch.cuda.synchronize()
    import numpy as np
    counts = np.concatenate([world.debug(f, "num_fluid_contacts").astype(np.int64) for f in fh])
    bits = int(world.debug(fh[0], "fluid_list_bits")[0]) if n else 32
    lbytes = list_bytes(counts, bits)
    out = args.out or tempfile.mkdtemp(prefix="profile_step_")
    os.makedirs(out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(out, "profile_step_%s.pt.trace.json" % args.config))
    st = world.stats()
    world.close()

    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or "k_" not in ev.name:
            continue
        k = kernel_key(ev.name)
        r = rows.setdefault(k, {"launches": 0, "us": 0.0})
        r["launches"] += 1
        r["us"] += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
    table = []
    for k, r in rows.items():
        ms = r["us"] / 1e3 / args.steps
        launches = r["launches"] / args.steps
        base = k.split("@")[0].split("<")[0]
        nbytes = BYTES.get(base)
        gbs = None
        if base in GATHER_OWN:
            nbytes = (GATHER_OWN[base] * n + lbytes) * launches
        elif nbytes is not None:
            nbytes = nbytes * n * launches
        if nbytes is not None and ms > 0:
            gbs = nbytes / (ms * 1e-3) / 1e9
        table.append({"phase": phase_of(k), "kernel": k, "launches_per_step": launches, "ms_per_step": ms,
                      "bytes_per_step": nbytes, "gb_per_s": gbs})
    order = {ph: i for i, (ph, _) in enumerate(PHASES)}
    order["other"] = len(PHASES)
    table.sort(key=lambda t: (order[t["phase"]], -t["ms_per_step"]))

    info = gpu_info()
    print("%s, %d fluid particles, %d profiled steps; card: %s, power limit %s W" %
          (args.config.upper(), n, args.steps, info.get("name"), info.get("power_limit_w")))
    print("step_ms (CUDA events, under the profiler): %s; iterations (div, press) last step: %d, %d" %
          (", ".join("%.3f" % s for s in step_ms), st["n_divergence_iter"], st["n_pressure_iter"]))
    print("fluid lists: %d-bit entries, %.1f contacts per particle, %.1f B per particle per pass" %
          (bits, counts.mean() if n else 0.0, lbytes / max(n, 1)))
    print("%-22s %-34s %8s %10s %10s %8s" % ("phase", "kernel", "launch/s", "ms/step", "MB/step", "GB/s"))
    tot = {}
    for t in table:
        tot[t["phase"]] = tot.get(t["phase"], 0.0) + t["ms_per_step"]
        print("%-22s %-34s %8.2f %10.4f %10s %8s" % (t["phase"], t["kernel"][:34], t["launches_per_step"], t["ms_per_step"],
              "-" if t["bytes_per_step"] is None else "%.1f" % (t["bytes_per_step"] / 1e6),
              "-" if t["gb_per_s"] is None else "%.0f" % t["gb_per_s"]))
    print("phase totals (ms/step): " + ", ".join("%s %.3f" % (ph, tot[ph]) for ph in sorted(tot, key=lambda p: order[p])))
    print("kernel total: %.3f ms/step" % sum(tot.values()))
    if args.json:
        with open(args.json, "w") as fh_:
            json.dump({"config": args.config, "particles": n, "gpu": info, "step_ms": step_ms, "list_bits": bits,
                       "list_bytes_per_pass": lbytes, "kernels": table}, fh_, indent=1)


if __name__ == "__main__":
    main()
