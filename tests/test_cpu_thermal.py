"""Heat transfer without a device: the float64 operator (tests/thermal_ref.py) on a lattice -- zero for a linear field, a constant
for |x|^2 --, the antisymmetric pair exchange and the conservation of sum m T, the C_op bound of the substep count on the lattice
and the squeezed block, the nu(T) law, the exported symbols, the refusals of the headless app and the slab driver, and the calls one
step issues in the class layer and the python engine with heat transfer on.  numpy + scipy only."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import ref64
import test_cpu_step_traces as ST
import thermal_ref as TR
from util import ROOT

R, SPACING, M0, RHO0, RHOB = 0.04, 0.02, 76.596750762082e-6, 1.0, 1.4


def _pairs(pos, mass=None, posB=None, massB=None):
    posB = np.zeros((0, 3)) if posB is None else posB
    massB = np.zeros(0) if massB is None else massB
    A = SimpleNamespace(posF=pos, massF=np.full(len(pos), M0) if mass is None else mass, csF=np.array([0, len(pos)]), posB=posB,
                        massB=massB, csB=np.array([0, len(posB)]), g=SimpleNamespace(ncells=1), R=R)
    return ref64.Pairs(A)


def _lattice(k=14):
    g = np.arange(k) * SPACING
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    c = pos.mean(0)
    return pos, np.all(np.abs(pos - c) < SPACING * (k / 2 - 2.5), 1), c


def test_lattice_laplacian():
    """interior of the lattice at the scenes' mass: the operator of a linear field is 0 (1e-9 of its terms) and of |x|^2 one constant,
    7.27 rather than 6 because the scenes' mass puts the lattice at 0.816 rho0 (W(0) = 0) -- the same factor scales alpha"""
    pos, inner, c = _lattice()
    P = _pairs(pos)
    lin = TR.conduction(P, pos @ np.array([1.0, -2.0, 3.0]), 1.0, RHO0, RHOB)
    assert np.abs(lin["value"][inner]).max() <= 1e-9 * lin["mag"][inner].max()
    q = TR.conduction(P, ((pos - c) ** 2).sum(1), 1.0, RHO0, RHOB)["value"][inner]
    assert np.ptp(q) <= 1e-9 * q.max()
    assert abs(q.mean() - 7.2725) < 1e-3, q.mean()


def test_pair_exchange_is_antisymmetric_and_conserves_heat():
    rng = np.random.default_rng(3)
    pos, _, _ = _lattice(8)
    pos = pos + rng.uniform(-0.004, 0.004, pos.shape)
    mass = M0 * rng.uniform(0.5, 2.0, len(pos))
    gb = np.arange(-2, 10) * SPACING
    x, z = np.meshgrid(gb, gb, indexing="ij")
    wall = np.stack([x.ravel(), np.full(x.size, -SPACING), z.ravel()], 1)
    P = _pairs(pos, mass, wall, np.full(len(wall), 2 * M0))
    cF, _, _ = TR.coefficients(P, 1e-3, RHO0, RHOB)
    flux = mass[P.iF] * cF                       # m_i c_ij must equal m_j c_ji
    key = {(i, j): f for i, j, f in zip(P.iF, P.jF, flux)}
    assert max(abs(f - key[(j, i)]) / abs(f) for (i, j), f in key.items() if f != 0) < 1e-12
    T = rng.uniform(0, 100, len(pos))
    dT = TR.conduction(P, T, 1e-3, RHO0, RHOB)["value"]       # adiabatic walls (h = 0)
    assert abs(np.dot(mass, dT)) <= 1e-12 * np.dot(mass, np.abs(dT))
    T1 = TR.run(P, T, 1e-3, RHO0, RHOB, 4e-3, 20)
    assert abs(np.dot(mass, T1) - np.dot(mass, T)) <= 1e-12 * np.dot(mass, T)


@pytest.mark.parametrize("scene", ["lattice", "squeezed"])
@pytest.mark.parametrize("h", [0.0, 1.0, 3.0])
def test_substeps_keep_the_maximum_principle(scene, h):
    """dt_k sum_j c_ij <= 1 for the substep count of sphk_heat_substeps (SPHK_HEAT_COP) at several alpha dt; the largest
    sum_j c_ij R^2 / alpha is 21.0 on the lattice and 79.1 in the block squeezed to 0.7 (2.9 times the density)"""
    pos, _, c = _lattice()
    if scene == "squeezed":
        pos = (pos - c) * 0.7 + c + np.random.default_rng(0).uniform(-0.0014, 0.0014, pos.shape)
    gb = np.arange(-2, 16) * SPACING
    x, z = np.meshgrid(gb, gb, indexing="ij")
    wall = np.stack([x.ravel(), np.full(x.size, pos[:, 1].min() - SPACING), z.ravel()], 1)
    P = _pairs(pos, None, wall, np.full(len(wall), M0 * RHOB))
    for alpha, dt in ((1e-4, 4e-3), (1e-2, 4e-3), (1.0, 1e-3)):
        cs = TR.conduction(P, np.zeros(P.n), alpha, RHO0, RHOB, None, [(0.0, h)])["csum"]
        k = TR.substeps(alpha, h, R, dt)
        assert (dt / k) * cs.max() <= 1.0, (alpha, dt, k, cs.max())


def test_viscosity_law():
    T = np.array([-1e30, -50.0, 0.0, 20.0, 25.0, 60.0, 1e30, np.nan])
    nu = TR.nu_of_t(T, 0.1, 0.05, 20.0, 0.01, 1.0)
    raw = 0.1 * np.exp(-0.05 * (T[1:6] - 20.0))
    assert np.allclose(nu[1:6], np.clip(raw, 0.01, 1.0), rtol=1e-15)
    assert nu[0] == 1.0 and nu[6] == 0.01 and nu[7] == 1.0
    assert nu[3] == 0.1


def test_exports():
    lib = os.path.join(ROOT, "cpp-fluid-particles_b200", "libsphk.so")
    if not os.path.exists(lib):
        pytest.skip("libsphk.so not built")
    if shutil.which("nm") is None:
        pytest.skip("nm not available")
    import subprocess
    syms = subprocess.run(["nm", "-D", lib], capture_output=True, text=True).stdout
    for name in ("sphk_heat_substeps", "sphk_heat_step", "sphk_heat_conduction", "sphk_heat_stats", "sphk_thermal_viscosity",
                 "sphk_thermal_viscosity_eval"):
        assert f" T {name}" in syms, name


def test_capi_names_and_slab_refusal(pkg):
    from cpp_fluid_particles_b200 import capi, slabs
    for name in ("sphk_heat_substeps", "sphk_heat_step", "sphk_heat_conduction", "sphk_heat_stats", "sphk_thermal_viscosity",
                 "sphk_thermal_viscosity_eval"):
        assert name in capi.SPHK_FUNCTIONS
    for name in ("sph_app_set_thermal", "sph_app_set_thermal_viscosity", "sph_app_upload_temperature", "sph_app_download_temperature",
                 "sph_app_thermal_stats"):
        assert name in capi.SPH_APP_FUNCTIONS
    assert C.sizeof(capi.Thermal) == 16 + 8 * capi.THERMAL_GROUPS
    s = object.__new__(slabs.SlabSystem)
    with pytest.raises(ValueError):
        s.thermal = dict(alpha=1.0)
    s.thermal = None
    with pytest.raises(ValueError):
        capi.thermal(dict(alpha=1.0, bodies=[(0.0, 0.0)] * 65))


def test_host_substeps_without_a_device(built):
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    k = C.c_int(0)
    for alpha, h, dt in ((1e-3, 0.0, 4e-3), (0.5, 2.0, 4e-3), (0.0, 0.0, 1.0)):
        t = capi.thermal(dict(alpha=alpha, wall=(10.0, h)))
        assert L.sphk_heat_substeps(C.byref(t), C.c_float(R), C.c_float(dt), C.byref(k)) == 0
        assert k.value == TR.substeps(float(np.float32(alpha)), h, float(np.float32(R)), float(np.float32(dt)))
    t = capi.thermal(dict(alpha=1.0))
    assert L.sphk_heat_substeps(C.byref(t), C.c_float(R), C.c_float(100.0), C.byref(k)) != 0     # above 65536 substeps
    t.groups[0].h = -1.0
    assert L.sphk_heat_substeps(C.byref(t), C.c_float(R), C.c_float(1e-3), C.byref(k)) != 0


@pytest.mark.parametrize("extra", [
    ["--heat", "1e-3"], ["--heat", "1e-3,0.01,20,5"], ["--heat", "1e-3,nan"], ["--heat", "x,0.01"], ["--heater", "50"],
    ["--wall-temp", "50"], ["--tap-temp", "50"], ["--thermal-viscosity", "0.1,0.05"], ["--heat", "1e-3,0.01", "--ranks", "2"],
    ["--heat", "1e-3,0.01", "--heater", "50", "--stir", "2"], ["--heat", "1e-3,0.01", "--heater", "50", "--float", "0.5"],
    ["--heat", "1e-3,0.01", "--tap-temp", "50"], ["--heat", "1e-3,0.01", "--wall-temp", "50,1,2"],
    ["--heat", "1e-3,0.01", "--thermal-viscosity", "0.1"], ["--heat", "1e-3,0.01", "--thermal-viscosity", "0.1,0.05,inf"],
    ["--heat", "1e-3,0.01", "--thermal-viscosity", "0.1,0.05", "--rheology", "hb:0.1,1,0.5"],
    ["--heat", "1e-3,0.01", "--thermal-viscosity", "0.1,0.05", "--implicit-viscosity", "0.1"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call"""
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


def test_python_refuses_a_rheology_with_a_thermal_viscosity():
    import pkgload
    pkgload.load()
    from cpp_fluid_particles_b200 import engine
    s = object.__new__(engine.SphkOps)
    s.thermal_viscosity = dict(nu_ref=0.1, e=0.0, nu_max=1.0)
    with pytest.raises(ValueError):
        s.rheology = dict(model="cross", nu0=0.1, nu_inf=0.01, lam=1.0, m=1.0, nu_max=0.1)
    s.thermal_viscosity = None
    s.rheology = dict(model="cross", nu0=0.1, nu_inf=0.01, lam=1.0, m=1.0, nu_max=0.1)
    with pytest.raises(ValueError):
        s.thermal_viscosity = dict(nu_ref=0.1, e=0.0, nu_max=1.0)


# ---- the class layer and the python engine issue the same calls with heat transfer on ----------------------------------------
# the implicit flag selects nu(T); not with a dynamic body, which refuses a wall factor > 0
THERMAL_CONFIGS = [c for c in ST.CONFIGS if not (c[4] and c[5])]
SPEC = dict(alpha=1e-3, beta=0.01, t_ref=20.0, wall=(60.0, 0.5))
NU_T = dict(nu_ref=1e-3, e=0.02, nu_max=0.1, wall_factor=1.0, tol=1e-4, max_iter=7)


@pytest.fixture(scope="module")
def thermal_traces(tmp_path_factory):
    d = tmp_path_factory.mktemp("thermal_traces")
    stub = d / "sphk_stub.cpp"
    stub.write_text(ST.stub_source(os.path.join(ROOT, "include", "sphk.h")))
    exe = str(d / "thermal_trace_driver")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    cmd = [cxx, "-std=c++17", "-O0", "-I" + os.path.join(ROOT, "include"), "-I" + ST.HOST, "-I/usr/local/cuda/include", "-o", exe,
           os.path.join(ST.HOST, "sph_api.cpp"), str(stub), os.path.join(ROOT, "tests", "thermal_trace_driver.cpp"),
           "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe] + [ST.config_id(c) for c in THERMAL_CONFIGS], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    traces = {}
    for line in r.stdout.splitlines():
        if line.startswith("TRACE "):
            _, key, *calls = line.split()
            traces[key] = calls
    assert sorted(traces) == sorted(ST.config_id(c) for c in THERMAL_CONFIGS), r.stdout[-3000:]
    return traces


@pytest.mark.parametrize("config", THERMAL_CONFIGS, ids=[ST.config_id(c) for c in THERMAL_CONFIGS])
def test_layers_issue_the_same_calls_with_heat_transfer(thermal_traces, config, monkeypatch):
    """permute, substeps, heat steps and (implicit flag) the nu(T) solve, in the same order and with the same halo kinds"""
    from cpp_fluid_particles_b200 import engine
    alloc = engine.SphkOps._alloc_solver_buffers

    def alloc_and_set(self, n):
        alloc(self, n)
        self.thermal = SPEC
        if config[4]:
            self.thermal_viscosity = NU_T
    monkeypatch.setattr(engine.SphkOps, "_alloc_solver_buffers", alloc_and_set)
    cpp = ST.compared(thermal_traces[ST.config_id(config)])
    py = ST.compared(ST.python_trace(config))
    assert "sphk_heat_step" in cpp and cpp.count("sphk_permute") >= 1
    assert ("sphk_thermal_viscosity" in cpp) == bool(config[4]) and "sphk_implicit_viscosity" not in cpp
    assert py == cpp
