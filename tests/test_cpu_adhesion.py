"""Fluid-solid adhesion without a device: the kernel A(r) of the float64 reference (tests/adhesion_ref.py), the reference on a flat
wall, the exported symbols and header constants, the refusals of the headless app and the slab driver, and the calls one step issues
in the class layer and the python engine with adhesion on.  numpy + scipy only."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import adhesion_ref as AR
import ref64
import test_cpu_step_traces as ST
from util import ROOT

R, SPACING, M0, RHO0, RHOB = 0.04, 0.02, 76.596750762082e-6, 1.0, 1.4


def test_kernel_band_ends_and_maximum():
    r = np.linspace(0.0, 1.5 * R, 300001)
    A = AR.kernel(r, R)
    assert np.all(A[(r <= 0.5 * R) | (r > R)] == 0.0)
    assert np.all(A[(r > 0.5 * R * (1 + 1e-9)) & (r < R * (1 - 1e-9))] > 0.0)
    assert AR.kernel(0.5 * R, R) == 0.0 and AR.kernel(R, R) == 0.0          # zero, and continuous, at both ends
    assert AR.kernel(0.5 * R * (1 + 1e-12), R) < 3e-3 * AR.kernel(0.75 * R, R)       # (r - R/2)^(1/4) towards 0
    assert AR.kernel(R * (1 - 1e-12), R) < 3e-3 * AR.kernel(0.75 * R, R)
    assert abs(r[np.argmax(A)] - 0.75 * R) <= r[1] - r[0]
    assert np.isclose(A.max(), 0.007 / R ** 3.25 * (R / 4) ** 0.25, rtol=1e-12)


def test_flat_wall_pulls_along_the_normal():
    """a fluid column over a flat wall lattice: a_i is along -y only, zero for particles beyond R of the wall, and the wetted count
    is the particles with a wall particle in the band"""
    g = np.arange(-6, 7) * SPACING
    x, z = np.meshgrid(g, g, indexing="ij")
    wall = np.stack([x.ravel(), np.zeros(x.size), z.ravel()], 1)
    ys = np.array([0.3, 0.6, 0.75, 0.9, 1.1, 1.6]) * R
    fluid = np.stack([np.zeros(ys.size), ys, np.zeros(ys.size)], 1)
    A = SimpleNamespace(posF=fluid, massF=np.full(ys.size, M0), csF=np.array([0, ys.size]), posB=wall,
                        massB=np.full(len(wall), M0 * RHOB), csB=np.array([0, len(wall)]), g=SimpleNamespace(ncells=1), R=R)
    P = ref64.Pairs(A)
    a, lo, hi = AR.accel(P, [150.0], RHO0, RHOB)
    v = a.value
    assert np.abs(v[:, [0, 2]]).max() <= 1e-12 * np.abs(v[:, 1]).max()
    assert np.all(v[:4, 1] < 0.0)                  # towards the wall
    assert np.all(v[4:] == 0.0)                    # beyond R of every wall particle
    assert lo == hi == 4
    b, _, _ = AR.accel(P, [0.0], RHO0, RHOB)
    assert np.all(b.value == 0.0)
    assert np.allclose(AR.accel(P, [300.0], RHO0, RHOB)[0].value, 2.0 * v, rtol=1e-14)


def test_reaction_balances_the_fluid():
    """sum m_i dt a_i + J = 0 and H about the centre, in the reference itself (one body, group 1)"""
    rng = np.random.default_rng(4)
    g = np.arange(-3, 4) * SPACING
    x, z = np.meshgrid(g, g, indexing="ij")
    plate = np.stack([x.ravel(), np.zeros(x.size), z.ravel()], 1)
    fluid = rng.uniform(-0.06, 0.06, (200, 3))
    mass = M0 * rng.uniform(0.5, 2.0, 200)
    A = SimpleNamespace(posF=fluid, massF=mass, csF=np.array([0, 200]), posB=plate, massB=np.full(len(plate), M0 * RHOB),
                        csB=np.array([0, len(plate)]), g=SimpleNamespace(ncells=1), R=R)
    P = ref64.Pairs(A)
    groups = np.ones(len(plate), np.int64)
    a, _, _ = AR.accel(P, [0.0, 120.0], RHO0, RHOB, groups)
    JH = AR.reaction(P, [0.0, 120.0], RHO0, RHOB, 0.004, mass, plate, groups, [[0.0, 0.0, 0.0]])
    dp = 0.004 * (mass[:, None] * a.value).sum(0)
    assert np.abs(dp).max() > 0
    assert np.allclose(dp + JH[0, :3], 0.0, atol=1e-12 * np.abs(dp).max())


def test_exports():
    lib = os.path.join(ROOT, "cpp-fluid-particles_b200", "libsphk.so")
    if not os.path.exists(lib):
        pytest.skip("libsphk.so not built")
    if shutil.which("nm") is None:
        pytest.skip("nm not available")
    syms = subprocess.run(["nm", "-D", lib], capture_output=True, text=True).stdout
    for name in ("sphk_adhesion", "sphk_adhesion_accel", "sphk_adhesion_stats"):
        assert f" T {name}" in syms, name


def test_header_constants_and_capi(pkg):
    from cpp_fluid_particles_b200 import capi, slabs
    hdr = open(os.path.join(ROOT, "include", "sphk.h")).read()
    assert "#define SPHK_ADHESION_GROUPS (1 + SPHK_BODY_LIMIT)" in hdr
    for name in ("sphk_adhesion", "sphk_adhesion_accel", "sphk_adhesion_stats"):
        assert name in capi.SPHK_FUNCTIONS
    for name in ("sph_app_set_adhesion", "sph_app_adhesion_stats"):
        assert name in capi.SPH_APP_FUNCTIONS
    assert capi.ADHESION_GROUPS == 65 and C.sizeof(capi.Adhesion) == 4 + 4 * capi.ADHESION_GROUPS
    a = capi.adhesion(dict(wall=150.0, bodies=[0.0, 90.0]))
    assert a.n_groups == 3 and list(a.beta[:4]) == [150.0, 0.0, 90.0, 0.0]
    with pytest.raises(ValueError):
        capi.adhesion(dict(wall=1.0, bodies=[0.0] * 65))
    with pytest.raises(ValueError):
        capi.adhesion(dict(walls=1.0))
    s = object.__new__(slabs.SlabSystem)
    with pytest.raises(ValueError):
        s.adhesion = dict(wall=150.0)
    s.adhesion = None


def test_python_refuses_bad_settings():
    import pkgload
    pkgload.load()
    from cpp_fluid_particles_b200 import engine
    s = object.__new__(engine.SphkOps)
    for bad in (dict(wall=-1.0), dict(wall=float("nan")), dict(wall=float("inf")), dict(wall=1.0, bodies=[1.0])):
        with pytest.raises(ValueError):
            s.adhesion = bad
    s.adhesion = dict(wall=150.0)
    assert s.adhesion == dict(wall=150.0)
    s.adhesion = None


@pytest.mark.parametrize("extra", [
    ["--adhesion", "-1"], ["--adhesion", "nan"], ["--adhesion", "x"], ["--adhesion", "100,-1"], ["--adhesion", "1,2,3"],
    ["--adhesion", "100", "--ranks", "2"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call"""
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


# ---- the class layer and the python engine issue the same calls with adhesion on ---------------------------------------------
SPEC, SPEC_BODY = dict(wall=150.0), dict(wall=150.0, bodies=[90.0])


@pytest.fixture(scope="module")
def adhesion_traces(tmp_path_factory):
    d = tmp_path_factory.mktemp("adhesion_traces")
    stub = d / "sphk_stub.cpp"
    stub.write_text(ST.stub_source(os.path.join(ROOT, "include", "sphk.h")))
    exe = str(d / "adhesion_trace_driver")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    cmd = [cxx, "-std=c++17", "-O0", "-I" + os.path.join(ROOT, "include"), "-I" + ST.HOST, "-I/usr/local/cuda/include", "-o", exe,
           os.path.join(ST.HOST, "sph_api.cpp"), str(stub), os.path.join(ROOT, "tests", "adhesion_trace_driver.cpp"),
           "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe] + [ST.config_id(c) for c in ST.CONFIGS], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    traces = {}
    for line in r.stdout.splitlines():
        if line.startswith("TRACE "):
            _, key, *calls = line.split()
            traces[key] = calls
    assert sorted(traces) == sorted(ST.config_id(c) for c in ST.CONFIGS), r.stdout[-3000:]
    return traces


@pytest.mark.parametrize("config", ST.CONFIGS, ids=[ST.config_id(c) for c in ST.CONFIGS])
def test_layers_issue_the_same_calls_with_adhesion(adhesion_traces, config, monkeypatch):
    """the adhesion sweep right after the viscosity / surface block, with the same halo kinds, in both layers"""
    from cpp_fluid_particles_b200 import engine
    alloc = engine.SphkOps._alloc_solver_buffers

    def alloc_and_set(self, n):
        alloc(self, n)
        self.n_bodies = 1 if config[5] else 0
        self.adhesion = SPEC_BODY if config[5] else SPEC
    monkeypatch.setattr(engine.SphkOps, "_alloc_solver_buffers", alloc_and_set)
    cpp = ST.compared(adhesion_traces[ST.config_id(config)])
    py = ST.compared(ST.python_trace(config))
    assert cpp.count("sphk_adhesion") == 1
    i = cpp.index("sphk_adhesion")
    assert cpp[i + 1] == "halo1"
    assert py == cpp
