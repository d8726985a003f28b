"""CPU checks of DynamicContactSampling: the float32 numpy restatement the GPU tests hold the device to
(salva_b200.contact_sampling) against the float64 projections and the float64 reference (oracle/ref64_colliders.py) on one
cuboid, and the ABI value."""
import os
import subprocess

import numpy as np

from oracle import ref64_colliders as C64
from salva_b200 import BODY_DYNAMIC, DynamicContactSampling
from salva_b200.contact_sampling import BALL, CAPSULE, CUBOID, contact_sample, project_local

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def proj64(kind, p, l):
    """The projection rules in float64: (proj, inside) per point."""
    l = np.asarray(l, np.float64)
    out, ins = np.empty_like(l), np.empty(len(l), bool)
    for i, x in enumerate(l):
        if kind == BALL:
            n = np.linalg.norm(x)
            ins[i] = n <= p[0]
            out[i] = x * (p[0] / n)
        elif kind == CUBOID:
            e = np.asarray(p[:3], np.float64)
            c = np.clip(x, -e, e)
            ins[i] = np.array_equal(c, x)
            if not ins[i]:
                out[i] = c
                continue
            best, bid, mins = -np.inf, 0, False
            for a in range(3):
                mp, pm = -e[a] - x[a], x[a] - e[a]
                if mp < pm:
                    if pm > best:
                        best, bid, mins = pm, a, False
                elif mp > best:
                    best, bid, mins = mp, a, True
            out[i] = x
            out[i][bid] = -e[bid] if mins else e[bid]
        else:
            c = np.array([0.0, np.clip(x[1], -p[0], p[0]), 0.0])
            d = x - c
            n = np.linalg.norm(d)
            ins[i] = n <= p[1]
            out[i] = c + (np.array([p[1], 0, 0]) if n == 0 else d * (p[1] / n))
    return out, ins


def _points(rng, scale, n=2000):
    return (rng.normal(0, scale, (n, 3))).astype(F32)


def test_projections_match_float64():
    rng = np.random.default_rng(0)
    cases = [(BALL, [0.3]), (CUBOID, [0.3, 0.1, 0.2]), (CAPSULE, [0.2, 0.1])]
    for kind, p in cases:
        pts = _points(rng, 0.3)
        edge = {BALL: [[0.3, 0, 0], [0, -0.3, 0], [0.3 * (1 + 1e-7), 0, 0]],
                CUBOID: [[0.3, 0.1, 0.2], [-0.3, 0.1, 0.0], [0.0, 0.0, 0.0], [0.1, 0.1 - 1e-7, 0.05], [0.2, 0.0, 0.1],
                         [0.29, 0.09, 0.19], [0.3, 0.05, 0.05]],
                CAPSULE: [[0.0, 0.1, 0.0], [0.0, 0.5, 0.0], [0.1, 0.2, 0.0], [0.0, -0.2, 0.1], [0.05, 0.0, 0.0]]}[kind]
        pts = np.concatenate([pts, np.asarray(edge, F32)])
        q, ins, valid = project_local(kind, p, pts)
        assert valid.all()
        q64, ins64 = proj64(kind, np.asarray(p, F32).astype(np.float64), pts)
        # on the surface (edges and corners included) inside or not is a matter of rounding: compare the projection only
        near = np.abs(np.linalg.norm(pts.astype(np.float64) - q64, axis=1)) <= 1e-6
        assert near.sum() >= 2, kind
        assert np.array_equal(ins[~near], ins64[~near]), kind
        assert np.abs(q - q64).max() <= 1e-6, kind
    q, _, valid = project_local(BALL, [0.3], np.zeros((1, 3), F32))  # the ball's centre: no projection
    assert not valid[0]
    q, ins, _ = project_local(CAPSULE, [0.2, 0.1], np.array([[0.0, 0.1, 0.0]], F32))  # on the axis: along local +x
    assert ins[0] and np.array_equal(q[0], np.array([0.1, 0.1, 0.0], F32))


def _scene():
    """Particles around a cuboid on a dynamic body, at every branch: deep inside, in the shell, beyond 1.5 h but in the AABB,
    moving towards and away from the surface."""
    rng = np.random.default_rng(5)
    pos = (rng.random((3000, 3)) * 1.2 - 0.6).astype(F32)
    vel = rng.normal(0, 2.0, pos.shape).astype(F32)
    col = dict(kind=CUBOID, params=[0.2, 0.1, 0.15], rotation=np.eye(3, dtype=F32), translation=np.array([0.01, -0.02, 0.03], F32),
               body=BODY_DYNAMIC, linvel=np.array([0.1, 0.2, 0.3], F32), angvel=np.array([1.0, -2.0, 0.5], F32),
               world_com=np.array([0.0, 0.05, 0.0], F32))
    return pos, vel, col


def test_restatement_matches_float64_and_every_mutant_is_flagged():
    """One cuboid on a dynamic body against the float64 reference (oracle/ref64_colliders.py); the scenes of several
    colliders of every shape are in test_ref64_colliders.py."""
    pos, vel, col = _scene()
    dt, h, r = 0.02, 0.1, 0.025
    p32, v32, s32 = contact_sample(pos, vel, [col], dt, h, r)
    assert np.any(p32 != pos), "the scene pushes"
    res = C64.contact64(pos, vel, [col], dt, h, r)
    worst = C64.check_restatement(res, p32, v32, s32)
    assert max(worst.values()) <= 1.0, worst
    assert res.excluded.sum() <= 0.01 * res.candidates
    for m in ("current_position", "current_dt", "local_point_velocity", "no_vn_gate", "no_margin", "no_cut", "aabb_not_loosened"):
        res = C64.contact64(pos, vel, [col], dt, h, r, dt_step=0.5 * dt, mutant=m)
        assert max(C64.check_restatement(res, p32, v32, s32).values()) > 1.0, m


def test_points_on_the_surface_are_sampled_without_a_push():
    """|dpt| <= f32::EPSILON (Unit::try_new_and_get fails): no push, and the sample is kept, at the projection."""
    col = dict(kind=CUBOID, params=[0.2, 0.1, 0.15], rotation=np.eye(3, dtype=F32), translation=np.zeros(3, F32), body=BODY_DYNAMIC,
               linvel=np.zeros(3, F32), angvel=np.zeros(3, F32), world_com=np.zeros(3, F32))
    pos = np.array([[0.2, 0.0, 0.0], [0.05, 0.1, -0.15], [0.2, 0.1, 0.15]], F32)  # a face, an edge, a corner
    vel = np.zeros_like(pos)
    branches = {}
    p2, v2, s = contact_sample(pos, vel, [col], 0.01, 0.1, 0.025, branches)
    assert np.array_equal(p2, pos) and np.array_equal(v2, vel)
    assert np.array_equal(s[0][0], pos)
    assert branches["on_surface"] == 3 and branches["pushed"] == 0
    res = C64.contact64(pos, vel, [col], 0.01, 0.1, 0.025)
    assert not res.excluded.any() and res.branches[CUBOID]["on_surface"] == 3
    assert np.array_equal(res.pos, pos) and np.array_equal(res.samples[0]["q"], pos)


def test_sampling_kind_matches_the_c_header(tmp_path):
    src = tmp_path / "kind.c"
    src.write_text('#include <stdio.h>\n#include "sph.h"\nint main(void) { printf("%d\\n", SPH_SAMPLING_CONTACT); return 0; }\n')
    exe = tmp_path / "kind"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = int(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout)
    assert got == DynamicContactSampling.kind == 1
