"""CPU-side checks of the boundary: the C-ABI libraries load and export every symbol the headers
declare; without a GPU the product fails loudly (no CPU fallback).  No compute calls here."""
import ctypes as C
import os
import re

import pytest

from util import ROOT


def _declared(header):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(sphk_[a-z_0-9]+|sph_app_[a-z_0-9]+)\s*\(", txt)))


def test_sphk_exports_every_declared_symbol(pkg, built):
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    names = _declared("sphk.h")
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert sorted(capi.SPHK_FUNCTIONS) == names, "capi.SPHK_FUNCTIONS out of sync with include/sphk.h"


def test_host_facade_exports_every_declared_symbol(pkg, built):
    from cpp_fluid_particles_b200 import capi
    L = capi.app_lib()
    names = [n for n in _declared("sph_app.h") if n != "sph_app_params"]
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert L.sph_app_engine() == b"b200-native"


def test_reference_facade_is_the_same_source(built):
    """The drop-in claim: ONE facade source, compiled against either header set."""
    mk = open(os.path.join(ROOT, "oracle", "ref_build", "Makefile")).read()
    assert "cpp-fluid-particles_b200/facade/sph_app.cpp" in mk
    src = open(os.path.join(ROOT, "cpp-fluid-particles_b200", "facade", "sph_app.cpp")).read()
    for inc in ("DArray.h", "Particles.h", "SPHParticles.h", "BaseSolver.h", "BasicSPHSolver.h", "DFSPHSolver.h",
                "PBDSolver.h", "SPHSystem.h"):
        assert f'#include "{inc}"' in src       # the reference's own include names (main.cpp:26-33)


def test_no_device_fails_loudly(pkg, built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    ctx = C.c_void_p()
    g = capi.SphkGrid(); g.cell_size[:] = [4, 4, 4]; g.cell_length = 0.1
    rc = L.sphk_create(C.byref(ctx), 8, 8, C.byref(g), None)
    assert rc == -2 and not ctx.value
    assert b"no CPU path" in L.sphk_error_string(rc)
    with pytest.raises(RuntimeError):
        capi.SphApp(pkg.scene.make_scene("mini"))


def test_product_never_imports_oracle():
    """oracle/ is test infrastructure: nothing under the package, include/ or pkgload may reference it."""
    bad = []
    for base in ("cpp-fluid-particles_b200", "include"):
        for dp, _, fs in os.walk(os.path.join(ROOT, base)):
            for f in fs:
                if f.endswith((".py", ".cpp", ".hpp", ".h", ".cu", ".cuh")):
                    txt = open(os.path.join(dp, f), errors="ignore").read()
                    if re.search(r"(from|import)\s+oracle|liboracle|oracle/sph_oracle", txt):
                        bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_mg_entry_points_validate_arguments(pkg, built):
    """The multi-GPU exchanges (csrc/sphk_mg.cu) reject bad arguments and, like sphk_create, refuse to run without a
    device -- no compute here."""
    import torch
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    ident = (C.c_ubyte * 128)()
    comm = C.c_void_p()
    assert L.sphk_mg_init(C.byref(comm), 3, 2, ident, None, C.c_longlong(0)) == -1      # rank >= world
    assert L.sphk_mg_init(None, 0, 1, ident, None, C.c_longlong(0)) == -1
    assert L.sphk_mg_halo(None, None, None, 0, None, 1, None) == -1
    assert L.sphk_mg_exchange_ints(None, None, None, None, None, 1) == -1
    assert L.sphk_mg_exchange_slices(None, 1, None, None, None, None, None, None, None) == -1
    assert L.sphk_mg_set_transport(None, 1) == -1
    assert L.sphk_mg_check(None, None) == -1
    # strays: block size arithmetic {4 header floats + capacity * sum(widths)} and argument validation
    w3 = (C.c_int * 3)(3, 3, 1)
    assert L.sphk_strays_block_floats(2048, 3, w3) == 4 + 2048 * 7
    assert L.sphk_strays_block_floats(8, 5, w3) == -1 and L.sphk_strays_block_floats(-1, 3, w3) == -1
    assert L.sphk_strays_collect(None, None, 0, 0, 3, None, w3, None, 8) == -1
    assert L.sphk_strays_append(None, None, 2, 8, 3, None, w3, 0) == -1
    assert L.sphk_mg_strays_route(None, None, None, None, 8, 3, None, w3, 0) == -1
    assert L.sphk_strays_counts(None, None, 2, 8, 3, w3, None) == -1
    L.sphk_mg_destroy(None)                                                             # no-op
    assert b"multi-GPU" in L.sphk_error_string(-6)
    if not torch.cuda.is_available():
        rc = L.sphk_mg_init(C.byref(comm), 0, 1, ident, None, C.c_longlong(0))
        assert rc in (-2, -6) and not comm.value      # no device (or no NCCL library): fails loudly, nothing created


def test_headless_cli_scene_matches_benchmark_scenes_and_fails_loudly(pkg, built, tmp_path):
    """app/sph_headless.cpp (the reference application without its window, SURVEY 8f-1): its C++ scene generator
    reproduces the python generator the benchmarks use bit for bit, and without a GPU it refuses to run."""
    import subprocess
    import numpy as np
    import torch
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    assert os.path.exists(cli)
    cases = [("config0", []),
             ("slabtest", ["--box", "2.0", "1.0", "1.0", "--block", "64", "24", "24", "--origin", "0.285", "0.105", "0.285"])]
    for name, args in cases:
        pre = str(tmp_path / name)
        r = subprocess.run([cli, "--emit-scene", pre] + args, capture_output=True, text=True, timeout=60)
        assert r.returncode == 0, r.stderr
        sc = pkg.scene.make_scene(name)
        assert f"{list(int(c) for c in sc.params.cell_size)}" in r.stdout
        fl = np.fromfile(pre + ".fluid.f32", np.float32).reshape(-1, 3)
        bd = np.fromfile(pre + ".boundary.f32", np.float32).reshape(-1, 3)
        assert np.array_equal(fl, sc.fluid) and np.array_equal(bd, sc.boundary), name
    if not torch.cuda.is_available():
        r = subprocess.run([cli, "--frames", "1"], capture_output=True, text=True, timeout=60)
        assert r.returncode == 3 and "no CPU path" in r.stderr
        # --ranks N: one forked rank per GPU (SlabSPHSystem); without devices every rank refuses and the launcher reports it
        r = subprocess.run([cli, "--frames", "1", "--ranks", "2"], capture_output=True, text=True, timeout=60)
        assert r.returncode == 3 and "no CPU path" in r.stderr      # (the first rank to fail ends the job)
    assert subprocess.run([cli, "--ranks", "2", "--rank", "1"], capture_output=True, timeout=60).returncode == 2   # needs --rendezvous
    assert subprocess.run([cli, "--solver", "nonsense"], capture_output=True, timeout=60).returncode == 2


def test_class_api_conformance_compiles_against_both_header_sets():
    """tests/api_conformance.cpp states the reference's public class API member by member (static_asserts).  It must
    compile against this repository's headers and -- where the reference sources exist (this container, not the GPU
    box) -- against the reference's own headers: same file, both engines."""
    import shutil
    import subprocess
    src = os.path.join(ROOT, "tests", "api_conformance.cpp")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    ours = [cxx, "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"),
            "-I" + os.path.join(ROOT, "cpp-fluid-particles_b200", "host"), "-I/usr/local/cuda/include", src]
    r = subprocess.run(ours, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    ref = "/root/reference/src"
    if os.path.isdir(ref):
        theirs = [cxx, "-std=c++17", "-fsyntax-only", "-fpermissive", "-w", "-DSPH_APP_REFERENCE_ENGINE",
                  "-I" + os.path.join(ROOT, "oracle", "ref_build"), "-I" + ref, "-I/usr/local/cuda/include", src]
        r = subprocess.run(theirs, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-3000:]
    # the assertions bite: a wrong signature is rejected
    bad = open(src).read().replace("float (SPHSystem::*)()", "double (SPHSystem::*)()")
    r = subprocess.run(ours[:-1] + ["-x", "c++", "-"], input=bad, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "float step()" in r.stderr


def test_tile_geometry_matches_the_library():
    """capi's tile-list constants size the buffers sphk_get_tile_lists copies into: they must be the C definitions."""
    from cpp_fluid_particles_b200 import capi
    txt = open(os.path.join(ROOT, "cpp-fluid-particles_b200", "csrc", "sphk_internal.cuh")).read()
    defs = {k: int(v) for k, v in re.findall(r"#define (SPHK_BLOCK|SPHK_TILE_WINS|SPHK_TILE_CAP)\s+(\d+)", txt)}
    assert defs == {"SPHK_BLOCK": capi.TILE_PARTICLES, "SPHK_TILE_WINS": capi.TILE_WINDOWS, "SPHK_TILE_CAP": capi.TILE_CAP}
