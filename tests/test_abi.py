"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/sph.h declares, and the product fails loudly (no CPU fallback) without a CUDA device."""
import ctypes as C
import os
import re

import pytest

from salva_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "sph.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sph_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_all_bound_and_exported():
    names = _declared_symbols()
    assert len(names) >= 20
    for path in (_lib.LIB_PATH, _lib.KERNELS_LIB_PATH):
        L = C.CDLL(path)
        for n in names:
            assert hasattr(L, n), "%s does not export %s" % (os.path.basename(path), n)
            assert n in _lib.SYMBOLS, "python binding misses %s" % n
    lean, full = C.CDLL(_lib.LIB_PATH), C.CDLL(_lib.KERNELS_LIB_PATH)
    lean.sph_version.restype = full.sph_version.restype = C.c_char_p
    assert b"poly6" in full.sph_version() and b"poly6" not in lean.sph_version()
    assert set(_lib.SYMBOLS) == set(names)


def test_struct_layouts_match_header():
    assert C.sizeof(_lib.WorldDesc) == 17 * 4
    assert C.sizeof(_lib.ForceDesc) == 4 + 8 * 4
    assert C.sizeof(_lib.StepStats) == 12 * 4 + 4 * 4 + 2 * 4 + 3 * 8 + 4 + 3 * 4 + 8 + 4 * 4


def test_ctypes_struct_sizes_match_a_c_compiler(tmp_path):
    """The python binding's struct layouts against gcc's view of include/sph.h (sizes and a few offsets)."""
    import subprocess
    src = tmp_path / "sizes.c"
    src.write_text('''#include <stdio.h>
#include <stddef.h>
#include "sph.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(sph_world_desc), sizeof(sph_force_desc), sizeof(sph_step_stats),
           sizeof(sph_host_force_ctx), sizeof(sph_boundary_view), sizeof(sph_shape), sizeof(sph_coupling_manager),
           offsetof(sph_host_force_ctx, ff_offsets), offsetof(sph_host_force_ctx, boundaries));
    return 0;
}
''')
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(_lib.WorldDesc), C.sizeof(_lib.ForceDesc), C.sizeof(_lib.StepStats), C.sizeof(_lib.HostForceCtx),
            C.sizeof(_lib.BoundaryView), C.sizeof(_lib.Shape), C.sizeof(_lib.CouplingManagerC),
            _lib.HostForceCtx.ff_offsets.offset, _lib.HostForceCtx.boundaries.offset]
    assert got == want


def test_product_does_not_import_the_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may import, link or execute anything under oracle/."""
    pat = re.compile(r"^\s*(from|import)\s+oracle\b|#include\s*[\"<].*oracle|liboracle|CDLL\(.*oracle", re.M)
    for dirpath, _, files in os.walk(os.path.join(ROOT, "salva_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".inl", ".h", ".hpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert not pat.search(src), "%s references the oracle" % os.path.join(dirpath, f)


def test_no_cpu_fallback_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from salva_b200 import LiquidWorld, SphError
    with pytest.raises(SphError) as e:
        LiquidWorld(particle_radius=0.05)
    assert e.value.status == 2  # SPH_ERR_CUDA


@pytest.mark.parametrize("solver, backend", [("dfsph", 1), ("iisph", 1), ("dfsph", 2)])
def test_gather_backend_other_than_0_is_refused(solver, backend):
    """gather_backend must be 0; the check runs before any device query, so it holds with or without a GPU."""
    from salva_b200 import DFSPHSolver, IISPHSolver, LiquidWorld, SphError
    with pytest.raises(SphError) as e:
        LiquidWorld(solver={"dfsph": DFSPHSolver, "iisph": IISPHSolver}[solver](), particle_radius=0.05, gather_backend=backend)
    assert e.value.status == 1  # SPH_ERR_INVALID


def test_every_entry_point_cites_the_reference_and_is_in_the_integration_guide():
    """include/sph.h declares the drop-in boundary: every entry point must appear in INTEGRATION.md (what it replaces in the
    reference), and the header itself must cite reference files (file.rs:line) next to the declarations."""
    header = open(os.path.join(ROOT, "include", "sph.h")).read()
    guide = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    missing = [s for s in _declared_symbols() if s not in guide]
    assert not missing, missing
    assert len(re.findall(r"[a-z_0-9]+\.rs:\d+", header)) >= 30
