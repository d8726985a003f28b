"""Times sph_world_sample_shape on three workloads: surface sampling of heightfield3's ground (41 x 41, r = 0.1) and of a
1000 x 1000 heightfield, and volume sampling of a cuboid into about 10M points.  Each call is bracketed by CUDA events
after warm-up calls; the call is synchronous, so the time covers the whole call: host set-up, the kernels, the sort
and the copy of the points to the host.  The float32 restatement on the host (oracle/ref64_sampling.py, numpy) is timed
on the same workloads for comparison (--no-host skips it on the two large ones).  Prints one JSON line with the card's
name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from salva_b200 import LiquidWorld  # noqa: E402
from salva_b200 import sampling as S  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "error": str(e)[:80]}


def ground():
    """heightfield3.rs:46-61: 3.0 on the rim, sin(i * 12 / 40) + cos(j * 12 / 40) inside."""
    n = 41
    i, j = np.meshgrid(np.arange(n, dtype=np.float32), np.arange(n, dtype=np.float32), indexing="ij")
    H = (np.sin(i * np.float32(12) / np.float32(40)) + np.cos(j * np.float32(12) / np.float32(40))).astype(np.float32)
    H[[0, -1], :] = 3.0
    H[:, [0, -1]] = 3.0
    return H


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-host", action="store_true")
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    big = np.cumsum(np.cumsum(rng.normal(0, 0.02, (1000, 1000)), 0), 1).astype(np.float32)
    big = (big - big.mean()) / (np.abs(big).max() + 1e-6) * 2.0
    r = 2.0 ** -7
    work = [("heightfield3_ground_surface", S.HeightField(ground(), (12.0, 1.0, 12.0)), 0.1, False),
            ("heightfield_1000x1000_surface", S.HeightField(big, (100.0, 4.0, 100.0)), 0.05, False),
            ("cuboid_10M_volume", S.Cuboid([215 * r, 216 * r, 217 * r]), r, True),
            ("cylinder_volume", S.Cylinder(1.0, 0.5), 0.005, True),
            ("cone_surface", S.Cone(1.0, 0.8), 0.002, False)]
    w = LiquidWorld(particle_radius=0.05)
    res = {"card": card(), "workloads": []}
    for name, shape, rad, vol in work:
        fn = S.shape_volume_ray_sample if vol else S.shape_surface_ray_sample
        pts = fn(w, shape, rad)
        for _ in range(2):
            fn(w, shape, rad)
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            fn(w, shape, rad)
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        row = {"workload": name, "points": int(len(pts)), "gpu_call_ms_median": float(np.median(ms)), "gpu_call_ms_min": float(min(ms))}
        # per-phase device time of one call: kernels and copies by name, from the profiler's CUDA activity
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            fn(w, shape, rad)
        phases = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                key = ("k_sample_rays<count>" if "k_sample_rays<false>" in ev.name else "k_sample_rays<fill>" if "k_sample_rays<true>" in ev.name
                       else "k_sample_unquantize" if "unquantize" in ev.name else "cub sort" if "RadixSort" in ev.name
                       else "cub unique" if "Select" in ev.name else "cub scan" if "Scan" in ev.name
                       else "memcpy " + ("DtoH" if "DtoH" in ev.name else "HtoD" if "HtoD" in ev.name else "other") if "emcpy" in ev.name else ev.name[:40])
                phases[key] = phases.get(key, 0.0) + ev.device_time_total / 1000.0
        row["phases_ms"] = {k: round(v, 4) for k, v in sorted(phases.items(), key=lambda kv: -kv[1])}
        if not a.no_host or name.startswith("heightfield3"):
            from oracle import ref64_sampling as R
            sh = (R.Shape(R.HEIGHTFIELD, heights=shape.heights, scale=shape.scale) if isinstance(shape, S.HeightField)
                  else R.Shape(shape.kind, shape.params))
            t = time.perf_counter()
            ref = R.sample(sh, rad, vol)
            row["host_f32_restatement_s"] = time.perf_counter() - t
            row["host_keys_decided"] = int(len(ref.keys))
        res["workloads"].append(row)
    w.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
