"""CPU checks of the collider coupling's float64 reference (oracle/ref64_colliders.py): the float32 restatement of contact
sampling the device is held to bit for bit (salva_b200.contact_sampling) meets its bounds on every scene the GPU checks step,
every plausible bug is flagged, exclusions stay rare, and the static pose and impulse references agree with numpy."""
import numpy as np
import pytest

from oracle import ref64_colliders as C64
from salva_b200.contact_sampling import contact_sample

F = np.float32


def _steps(name, mutant=None, steps=None):
    """Steps a scene through the float32 restatement (P' = P + v dt after each pass, as the device with the solver's
    iterations at zero), checking each pass against the reference fed the same input."""
    sc = C64.SCENES[name]()
    pos = np.concatenate([f["positions"] for f in sc["fluids"]])
    vel = np.concatenate([f["velocities"] for f in sc["fluids"]])
    h = float(F(sc["radius"]) * F(2) * F(2))
    lag, worst, excluded, candidates, branches = 0.0, {}, 0, 0, {}
    for k in range(steps or sc["steps"]):
        dt = C64.DTS[k % len(C64.DTS)]
        cols = C64.colliders_at(sc, k)
        p32, v32, s32 = contact_sample(pos, vel, cols, lag, h, sc["radius"])
        res = C64.contact64(pos, vel, cols, lag, h, sc["radius"], dt_step=dt, mutant=mutant)
        for key, val in C64.check_restatement(res, p32, v32, s32).items():
            worst[key] = max(worst.get(key, 0.0), val)
        excluded += int(res.excluded.sum())
        candidates += res.candidates
        for kind, d in res.branches.items():
            for b, n in d.items():
                branches.setdefault(kind, {}).setdefault(b, 0)
                branches[kind][b] += n
        pos, vel, lag = (p32 + v32 * F(dt)).astype(F), v32, dt
    return worst, excluded, candidates, branches


@pytest.mark.parametrize("name", sorted(C64.SCENES))
def test_restatement_meets_the_float64_bounds(name):
    worst, excluded, candidates, _ = _steps(name)
    print("\nREF64 colliders restatement %s worst %s excluded %d of %d" % (name, {k: round(v, 4) for k, v in worst.items()}, excluded, candidates))
    assert max(worst.values()) <= 1.0, worst
    assert excluded <= 0.01 * candidates, (excluded, candidates)


def test_every_branch_is_reached_for_each_shape():
    _, _, _, br = _steps("overlap")
    for kind in (C64.BALL, C64.CUBOID, C64.CAPSULE):
        for b in ("pushed", "shell", "beyond", "prediction_outside", "cell_outside", "on_surface"):
            assert br[kind][b] > 0, (kind, b, br[kind])
    assert br[C64.BALL]["ball_centre"] > 0 and br[C64.CAPSULE]["capsule_axis"] > 0


def test_three_colliders_process_one_particle():
    sc = C64.SCENES["overlap"]()
    res = C64.run_reference(sc)[0]
    common = set(res.processed[0].tolist()) & set(res.processed[1].tolist()) & set(res.processed[2].tolist())
    assert common


@pytest.mark.parametrize("mutant", C64.CONTACT_MUTANTS)
def test_every_contact_mutant_is_flagged(mutant):
    worst, _, _, _ = _steps("overlap", mutant, steps=3)
    print("\nREF64 colliders mutant %s worst %s" % (mutant, worst))
    assert max(worst.values()) > 1.0, (mutant, worst)


def _static_f32(local, col):
    """k_collider_static's float32 expression: rot * local + t summed left to right, the velocity at the LOCAL point."""
    R, t = np.asarray(col["rotation"], F), np.asarray(col["translation"], F)
    x = np.stack([((R[a, 0] * local[:, 0] + R[a, 1] * local[:, 1]) + R[a, 2] * local[:, 2]) + t[a] for a in range(3)], axis=1).astype(F)
    lv, w, c = (np.asarray(col[k], F) for k in ("linvel", "angvel", "world_com"))
    d = local - c
    v = np.stack([lv[0] + (w[1] * d[:, 2] - w[2] * d[:, 1]), lv[1] + (w[2] * d[:, 0] - w[0] * d[:, 2]),
                  lv[2] + (w[0] * d[:, 1] - w[1] * d[:, 0])], axis=1).astype(F)
    return x, v


def test_static_pose_against_float32_and_the_world_point_mutant():
    rng = np.random.default_rng(2)
    local = rng.normal(0, 0.3, (500, 3)).astype(F)
    col = C64._state((0.7, -0.2, 1.3), C64.rot(0.4, -1.1, 2.0), C64.BODY_DYNAMIC, (0.5, -1, 2), (3, -2, 1), (0.6, -0.1, 1.2))
    x32, v32 = _static_f32(local, col)
    x, ex, v, ev = C64.static64(local, col)
    assert C64.ratio(x32, x, ex).max() <= 1.0 and C64.ratio(v32, v, ev).max() <= 1.0
    _, _, vm, evm = C64.static64(local, col, mutant="world_point_velocity")
    assert C64.ratio(v32, vm, evm).max() > 1.0


def _impulse_entries(rng):
    """Three colliders on boundary slots 2, 3 (adjacent, both dynamic) and 5 (fixed), collider slots 1, 0, 4."""
    out = []
    for slot, bslot, body in ((1, 2, C64.BODY_DYNAMIC), (0, 3, C64.BODY_DYNAMIC), (4, 5, C64.BODY_FIXED)):
        x = (rng.normal(0, 0.2, (700, 3)) + np.array([0.5, 0.3, 0.5])).astype(F)
        f = rng.normal(0, 1.0, (700, 3)).astype(F) + F(0.02)
        out.append(dict(slot=slot, bslot=bslot, body=body, translation=np.array([0.5, 0.3, 0.5], F),
                        world_com=np.array([0.65, 0.1, 0.4], F), positions=x, forces=f))
    return out


def _impulse_f32(e, dt, rng):
    """The kernel's per-term float32 expression, summed in float32 in a random order."""
    f = e["forces"] * F(dt)
    r = e["positions"] - e["world_com"]
    ang = np.stack([r[:, 1] * f[:, 2] - r[:, 2] * f[:, 1], r[:, 2] * f[:, 0] - r[:, 0] * f[:, 2], r[:, 0] * f[:, 1] - r[:, 1] * f[:, 0]], axis=1)
    o = rng.permutation(len(f))
    lin, an = np.zeros(3, F), np.zeros(3, F)
    for i in o:
        lin = (lin + f[i]).astype(F)
        an = (an + ang[i]).astype(F)
    return lin, an


def test_impulse_reference_against_float32_sums_and_every_mutant_is_flagged():
    rng = np.random.default_rng(9)
    entries = _impulse_entries(rng)
    dt, dt_prev = 0.008, 0.004
    got = {e["slot"]: (_impulse_f32(e, dt, rng) if e["body"] == C64.BODY_DYNAMIC else (np.zeros(3), np.zeros(3))) for e in entries}
    nb = sum(len(e["forces"]) for e in entries)

    def worst(ref):
        return max(max(float(C64.ratio(got[s][0], lin, el).max()), float(C64.ratio(got[s][1], ang, ea).max()))
                   for s, (lin, ang, el, ea) in ref.items())
    assert worst(C64.impulse64(entries, dt, dt_prev, nb)) <= 1.0
    for m in C64.IMPULSE_MUTANTS:
        assert worst(C64.impulse64(entries, dt, dt_prev, nb, mutant=m)) > 1.0, m
