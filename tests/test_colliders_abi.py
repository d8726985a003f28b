"""CPU-side checks of the collider coupling ABI (include/sph.h sph_collider_*): the ctypes layout of sph_collider_state
against gcc, and the numpy restatement the GPU tests pose sample points with."""
import ctypes as C
import os
import subprocess

import numpy as np

from salva_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_collider_state_layout_matches_a_c_compiler(tmp_path):
    src = tmp_path / "collider.c"
    src.write_text('''#include <stdio.h>
#include <stddef.h>
#include "sph.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %d %d %d %d\\n", sizeof(sph_collider_state), offsetof(sph_collider_state, rotation_rowmajor),
           offsetof(sph_collider_state, body), offsetof(sph_collider_state, angvel), offsetof(sph_collider_state, world_com),
           SPH_SAMPLING_STATIC, SPH_BODY_NONE, SPH_BODY_FIXED, SPH_BODY_DYNAMIC);
    return 0;
}
''')
    exe = tmp_path / "collider"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.ColliderState
    from salva_b200 import BODY_DYNAMIC, BODY_FIXED, BODY_NONE, StaticSampling
    assert got == [C.sizeof(S), S.rotation_rowmajor.offset, S.body.offset, S.angvel.offset, S.world_com.offset,
                   StaticSampling.kind, BODY_NONE, BODY_FIXED, BODY_DYNAMIC]


def test_pose_restatement_is_the_isometry():
    """The float32 restatement of k_collider_static agrees with a float64 isometry and with the reference's velocity at the
    local point (fluids_pipeline.rs:183) to rounding."""
    from test_gpu_colliders import local_velocity, pose_points, rot_zx
    rng = np.random.default_rng(1)
    local = rng.uniform(-1, 1, (100, 3)).astype(np.float32)
    R, t = rot_zx(0.7), np.array([0.5, -2.0, 3.0], np.float32)
    want = local.astype(np.float64) @ R.astype(np.float64).T + t
    assert np.abs(pose_points(local, R, t) - want).max() < 1e-5
    lv, w, c = np.array([1.0, 2.0, 3.0]), np.array([0.5, -1.0, 2.0]), np.array([0.1, 0.2, -0.3])
    want_v = lv + np.cross(w, local.astype(np.float64) - c)
    assert np.abs(local_velocity(local, lv, w, c) - want_v).max() < 1e-5
