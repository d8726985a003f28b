"""Step time of a heightfield ground coupled by DynamicContactSampling on the device, against the same ground coupled by
StaticSampling (its surface ray-sampled at r / 1.5, as heightfield3.rs does) and against the numpy restatement run as a host
CouplingManager (salva_b200.contact_sampling.ContactSamplingHook through step_with_coupling).

The scene is heightfield3.rs: a 15^3 block thrown at 10 m/s onto a fixed 12 m x 12 m heightfield (3.0 on the rim,
sin(x) + cos(z) inside), at heightfield3's 41 x 41 heights and on a fine 513 x 513 field over the same 12 m.  The variants
of a scene are stepped alternately in one process; each evolves on its own.  The card, its power limit and SM clock are
read in the same run.  Timing starts once the block has landed.  Prints one JSON line per scene: median step ms (CUDA events), median wall ms and kernels per step,
and, from a separate torch.profiler run of the device variant, k_contact_sample's time per step and per sample.

    python tools/bench_heightfield_contact.py --steps 30 --warmup 60
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_contact_sampling import CountingHook, card, run  # noqa: E402
from salva_b200 import BODY_FIXED, DFSPHSolver, DynamicContactSampling, LiquidWorld, StaticSampling, scenes  # noqa: E402
from salva_b200.sampling import HeightField, shape_surface_ray_sample  # noqa: E402

F32 = np.float32
R, DT, GRAVITY = 0.15, 1.0 / 200.0, (0.0, -9.81, 0.0)
FIXED = dict(translation=np.zeros(3, F32), rotation=np.eye(3, dtype=F32), body=BODY_FIXED)


def ground_heights(n):
    """heightfield3.rs:46-61 on an n x n grid over 12 m: 3.0 on the rim, sin(x) + cos(z) inside."""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    h = (np.sin((i * F32(12.0) / F32(n - 1)).astype(F32)) + np.cos((j * F32(12.0) / F32(n - 1)).astype(F32))).astype(F32)
    h[[0, -1], :] = 3.0
    h[:, [0, -1]] = 3.0
    return h


def make_world():
    w = LiquidWorld(DFSPHSolver(), particle_radius=R, smoothing_factor=2.0)
    pts = scenes.cube_fluid(15, 15, 15, F32(R))
    pts[:, 1] += F32(1.0) + F32(15) * F32(R) * F32(2.0)  # heightfield3.rs:33-37
    fh = w.add_fluid(pts, velocities=np.tile(np.array([0.0, -10.0, 0.0], F32), (len(pts), 1)), density0=1000.0)
    w.push_force(fh, *scenes.artificial_viscosity(1.0, 0.0))
    return w, fh


def variants(n, warmup):
    """The three variants after `warmup` steps of the device and StaticSampling worlds; the numpy hook's world starts from
    the device world's state then (a snapshot), so its slow steps are all timed on a landed block."""
    ground = HeightField(ground_heights(n), (12.0, 1.0, 12.0))
    dev, _ = make_world()
    c = dev.register_coupling(dev.add_boundary(np.zeros((0, 3), F32)), DynamicContactSampling(ground))
    dev.set_collider_state(c, body=BODY_FIXED)
    static, _ = make_world()
    samples = shape_surface_ray_sample(static, ground, F32(R) / F32(1.5))
    sc = static.register_coupling(static.add_boundary(np.zeros((0, 3), F32)), StaticSampling(samples))
    static.set_collider_state(sc, body=BODY_FIXED)
    host, hf = make_world()
    hook = CountingHook([hf], [(host.add_boundary(np.zeros((0, 3), F32)), dict(kind=4, params=(), heights=ground.heights, scale=ground.scale,
                                                                                  **FIXED))])

    for _ in range(warmup):
        dev.step(DT, GRAVITY)
        static.step(DT, GRAVITY)
    host.restore(dev.snapshot())

    def host_step():
        before = hook.calls
        host.step_with_coupling(DT, GRAVITY, hook)
        assert hook.calls == before + 1, "the host hook failed"  # exceptions inside the callback do not propagate

    v = {"device_contact": (dev, lambda i: (lambda: dev.step(DT, GRAVITY))),
         "static_sampling": (static, lambda i: (lambda: static.step(DT, GRAVITY))),
         "numpy_hook": (host, lambda i: host_step)}
    return v, len(samples)


def profile_contact(n, steps, warmup):
    """k_contact_sample's CUDA time per step and per sample of the device variant, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    w, _ = make_world()
    b = w.add_boundary(np.zeros((0, 3), F32))
    c = w.register_coupling(b, DynamicContactSampling(HeightField(ground_heights(n), (12.0, 1.0, 12.0))))
    w.set_collider_state(c, body=BODY_FIXED)
    for _ in range(warmup):
        w.step(DT, GRAVITY)
    samples = 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            w.step(DT, GRAVITY)
            samples += len(w.read_boundary_particles(b)[0])
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_contact_sample" in e.key)
    return dict(k_contact_sample_us_per_step=round(us / steps, 2), samples_per_step=samples // steps,
                k_contact_sample_ns_per_sample=round(1e3 * us / max(samples, 1), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per variant (the numpy hook takes seconds per step)")
    ap.add_argument("--warmup", type=int, default=60, help="steps before timing: the block lands from step 9 on")
    ap.add_argument("--sizes", default="41,513")
    a = ap.parse_args()
    for n in (int(s) for s in a.sizes.split(",")):
        gpu = card()
        v, nstatic = variants(n, a.warmup)
        out = run(v, DT, GRAVITY, a.steps, 2)
        print(json.dumps(dict(scene="heightfield3 ground %d x %d" % (n, n), gpu=gpu, static_samples=nstatic, **out,
                              device_kernel=profile_contact(n, 20, a.warmup))), flush=True)
    print(json.dumps(dict(gpu_after=card())))


if __name__ == "__main__":
    main()
