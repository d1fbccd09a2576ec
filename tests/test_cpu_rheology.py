"""Non-Newtonian viscosity without a device: the float64 reference (tests/rheology_ref.py) against closed forms -- the corrected
velocity gradient of a linear field, the shear rate of simple shear, the two models against their formulas over a grid of shear
rates from 0 through subnormals to 1e30 with both clamps -- the exported symbols, the refusals of the headless app and the slab
driver, and the calls one step issues in the class layer and the python engine with a rheology set.  numpy + scipy only."""
import ctypes as C
import math
import os
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import implicit_visc_ref as IV
import ref64
import rheology_ref as RR
import test_cpu_step_traces as ST
from util import ROOT

R, SPACING, M0, RHO0, RHOB = 0.04, 0.02, 76.596750762082e-6, 1.0, 1.4


def _pairs(pos, posB, mass, massB):
    A = SimpleNamespace(posF=pos, massF=mass, csF=np.array([0, pos.shape[0]]), posB=posB, massB=massB,
                        csB=np.array([0, posB.shape[0]]), g=SimpleNamespace(ncells=1), R=R)
    return ref64.Pairs(A)


def _scene(seed=1, k=8):
    """a jittered fluid block resting on a wall (two boundary layers), random masses: bulk, free surface, edges, corners and the
    wall side"""
    rng = np.random.default_rng(seed)
    g = np.arange(k) * SPACING + 0.1
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + rng.uniform(-0.004, 0.004, (k ** 3, 3))
    gb = np.arange(-2, k + 2) * SPACING + 0.1
    x, z = np.meshgrid(gb, gb, indexing="ij")
    wall = np.concatenate([np.stack([x.ravel(), np.full(x.size, 0.1 - d * SPACING), z.ravel()], 1) for d in (1, 2)])
    mass = M0 * rng.uniform(0.5, 2.0, pos.shape[0])
    massB = M0 * rng.uniform(1.0, 3.0, wall.shape[0])
    return pos, wall, mass, massB


# ---- 1. closed forms of the shear sweep -----------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_corrected_gradient_of_a_linear_field_is_exact(beta):
    """v = A x + b (on the walls too): grad v_i = A for every particle whose M_i passes the conditioning test -- the bulk, the free
    surface, edges, corners and the particles next to the wall"""
    pos, wall, mass, massB = _scene()
    P = _pairs(pos, wall, mass, massB)
    A = np.random.default_rng(5).standard_normal((3, 3))
    b = np.array([0.3, -0.2, 0.1])
    s = RR.shear(P, pos @ A.T + b, wall @ A.T + b, beta, RHO0, RHOB)
    ok = s["flag"] == 0
    nb = np.bincount(P.iF, minlength=P.n)
    assert ok.mean() > 0.95, ok.mean()
    assert (ok & (nb < 0.5 * nb.max())).sum() > 20, "no surface particle was corrected"
    err = np.abs(s["grad"][ok] - A[None]).max()
    assert err <= 1e-9 * np.abs(A).max(), err
    E = 0.5 * (A + A.T)
    assert np.allclose(s["gamma"][ok], np.sqrt(2.0 * (E * E).sum()), rtol=1e-9)


def test_scalar_normalisation_is_off_where_the_support_is_one_sided():
    """what the correction is for: with G_i 3 / tr M_i alone the gradient of a linear field is off by tens of percent at the free
    surface (printed: also in the bulk of the jittered block)"""
    pos, wall, mass, massB = _scene()
    P = _pairs(pos, wall, mass, massB)
    A = np.diag([1.0, 0.0, 0.0])
    s = RR.shear(P, pos @ A.T, wall @ A.T, 0.0, RHO0, RHOB)
    v = pos @ A.T
    G = RR._outer_sum_full(P.n, P.iF, v[P.jF] - v[P.iF], (P.mF / RHO0 * IV.grad_factor(P.rF, P.R)[0])[:, None] * P.dF)
    scalar = G * (3.0 / s["tr"])[:, None, None]
    err = np.abs(scalar[:, 0, 0] - 1.0)
    nb = np.bincount(P.iF, minlength=P.n)
    bulk, surf = nb >= 0.95 * nb.max(), nb < 0.6 * nb.max()
    print(f"\nscalar-normalised d vx / dx of vx = x: bulk mean error {err[bulk].mean():.3f}, surface mean error {err[surf].mean():.3f}")
    assert err[surf].mean() > 0.1


@pytest.mark.parametrize("gamma", [-3.0, 0.7, 25.0])
def test_simple_shear_gives_the_shear_rate(gamma):
    pos, wall, mass, massB = _scene(seed=2)
    P = _pairs(pos, wall, mass, massB)
    A = np.zeros((3, 3))
    A[0, 1] = gamma
    s = RR.shear(P, pos @ A.T, wall @ A.T, 1.0, RHO0, RHOB)
    ok = s["flag"] == 0
    assert np.allclose(s["gamma"][ok], abs(gamma), rtol=1e-9)


def test_few_neighbours_fall_back_to_the_scalar_normalisation():
    """a line of particles: M_i has rank 1, the conditioning test fails and the scalar normalisation is used"""
    pos = np.stack([0.1 + np.arange(6) * 0.015, np.full(6, 0.2), np.full(6, 0.2)], 1)
    P = _pairs(pos, np.zeros((0, 3)), np.full(6, M0), np.zeros(0))
    s = RR.shear(P, pos * 0.0 + np.array([1.0, 0.0, 0.0]), np.zeros((0, 3)), 0.0, RHO0, RHOB)
    assert np.all(s["flag"] == 1) and np.all(s["gamma"] == 0.0)
    iso = RR.shear(P, np.zeros((6, 3)), np.zeros((0, 3)), 0.0, RHO0, RHOB)
    assert np.all(iso["flag"] == 1)


# ---- 2. the models ----------------------------------------------------------------------------------------------------------
GRID = [0.0, 1e-45, 1e-38, 1e-30, 1e-10, 1e-3, 0.1, 1.0, 7.5, 1e3, 1e10, 1e30]


def _cross(p, g):
    nu0, nu_inf, lam, m = p
    return nu_inf + (nu0 - nu_inf) / (1.0 + (lam * g) ** m)


def _hb(p, g):
    K, n, tau, mr = p
    power = K * g ** (n - 1.0) if K > 0 and (g > 0 or n >= 1) else (math.inf if K > 0 else 0.0)
    if K > 0 and g == 0 and n == 1:
        power = K
    yield_ = tau * mr if g == 0 else tau * (1.0 - math.exp(-mr * g)) / g if mr * g > 1e-8 else tau * mr * (1.0 - 0.5 * mr * g)
    return power + yield_


@pytest.mark.parametrize("model,params", [
    (RR.CROSS, (0.5, 0.01, 2.0, 0.8)),      # shear-thinning
    (RR.CROSS, (0.05, 0.05, 3.0, 1.0)),     # Newtonian
    (RR.CROSS, (0.01, 0.3, 0.5, 2.0)),      # thickening in the Cross form
    (RR.HB, (0.02, 1.0, 0.5, 1000.0)),      # Bingham
    (RR.HB, (0.1, 0.4, 0.0, 1000.0)),       # power law, thinning
    (RR.HB, (0.1, 1.6, 0.0, 1000.0)),       # power law, thickening
    (RR.HB, (0.0, 1.0, 2.0, 50.0)),         # pure yield stress
])
def test_models_against_their_formulas(model, params):
    nu_min, nu_max = 1e-4, 3.0
    g = np.array(GRID)
    nu, at = RR.model_nu(model, params, nu_min, nu_max, g)
    for k, x in enumerate(GRID):
        raw = _cross(params, x) if model == RR.CROSS else _hb(params, x)
        want = nu_max if not raw < nu_max else max(raw, nu_min)
        assert nu[k] == pytest.approx(want, rel=1e-12, abs=0), (x, nu[k], want)
        assert bool(at[k]) == (not raw < nu_max)
    if model == RR.HB and params[2] > 0:
        lim = params[2] * params[3] + (params[0] if params[1] == 1.0 else 0.0)
        assert RR.model_nu(model, params, 0.0, 1e9, np.array([0.0]))[0][0] == pytest.approx(lim, rel=1e-15)
        assert RR.model_nu(model, params, 0.0, 1e9, np.array([1e-300]))[0][0] == pytest.approx(lim, rel=1e-12)


def test_clamps_and_nan():
    nu, at = RR.model_nu(RR.HB, (0.1, 0.4, 0.0, 1000.0), 0.02, 0.5, np.array([0.0, 1e-30, 1.0, 1e30, np.nan]))
    assert nu[0] == 0.5 and at[0]             # n < 1: K 0^(n-1) = inf -> nu_max
    assert nu[1] == 0.5 and at[1]
    assert nu[2] == pytest.approx(0.1) and not at[2]
    assert nu[3] == 0.02 and not at[3]        # nu_min
    assert nu[4] == 0.5 and at[4]             # a NaN rate lands on nu_max


# ---- 3. exports, refusals ---------------------------------------------------------------------------------------------------
NEW_SPHK = ("sphk_rheology_work_floats", "sphk_non_newtonian_viscosity", "sphk_non_newtonian_stats", "sphk_shear_rate",
            "sphk_rheology_eval", "sphk_visc_field_setup", "sphk_visc_field_matvec")
NEW_APP = ("sph_app_set_rheology", "sph_app_rheology_stats", "sph_app_download_viscosity")


def test_exported_symbols_and_validation_without_a_device(built):
    from cpp_fluid_particles_b200 import capi
    L = C.CDLL(capi.LIBSPHK)
    for name in NEW_SPHK:
        assert hasattr(L, name), name
        assert name in capi.SPHK_FUNCTIONS
    H = C.CDLL(capi.LIBHOST, mode=C.RTLD_LOCAL)
    for name in NEW_APP:
        assert hasattr(H, name), name
        assert name in capi.SPH_APP_FUNCTIONS
    L.sphk_rheology_work_floats.restype = C.c_longlong
    assert L.sphk_rheology_work_floats(C.c_int(1000)) == 64 + 6 * 1024 + 22 * 1000
    assert L.sphk_rheology_work_floats(C.c_int(-1)) < 0
    assert C.sizeof(capi.Rheology) == 36
    r = capi.rheology(dict(model="cross", nu0=0.1, nu_inf=0.01, lam=1.0, m=1.0, nu_max=0.1))
    INVALID = -1
    f = C.c_float
    assert L.sphk_non_newtonian_viscosity(None, None, None, None, C.byref(r), f(0), f(0.004), f(1), f(1.4), f(1e-4), C.c_int(10)) == INVALID
    assert L.sphk_rheology_eval(None, C.byref(r), None, None, C.c_int(1)) == INVALID
    assert L.sphk_non_newtonian_stats(None, None, None, None, None, None, None) == INVALID
    for bad in (dict(model="power"), dict(model="cross", nu0=0.1), dict(model="hb", k=1.0, n=1.0, tau_y=1.0),
                dict(model="hb", k=1.0, n=1.0, tau_y=1.0, nu_max=1.0, colour="red")):
        with pytest.raises(ValueError):
            capi.rheology(bad)
    h = capi.rheology(dict(model="hb", k=0.02, n=1.0, tau_y=0.5, nu_max=2.0))
    assert h.model == 2 and list(h.params)[:4] == [pytest.approx(0.02), 1.0, 0.5, 1000.0] and h.nu_max == 2.0


def test_slab_system_refuses_a_rheology(pkg):
    from cpp_fluid_particles_b200 import slabs
    obj = object.__new__(slabs.SlabSystem)
    obj.rheology = None
    with pytest.raises(ValueError):
        obj.rheology = dict(model="cross", nu0=0.1, nu_inf=0.01, lam=1.0, m=1.0, nu_max=0.1)
    assert obj.rheology is None


@pytest.mark.parametrize("extra", [
    ["--rheology", "cross:0.1,0.01,1"], ["--rheology", "cross:0.1,0.01,1,nan"], ["--rheology", "bingham:1,1,1"],
    ["--rheology", "hb:0.1,1"], ["--rheology", "hb:0.1,1,x"], ["--rheology", "hb:0.1,1,0.5", "--ranks", "2"],
    ["--rheology", "hb:0.1,1,0.5", "--implicit-viscosity", "0.1"], ["--rheology", "hb:0.1,1,0.5", "--no-slip", "--float", "0.5"],
    ["--no-slip"], ["--rheology-max", "2"], ["--rheology", "cross:0.1,0.01,1,1", "--rheology-max", "inf"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call"""
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


# ---- 4. the class layer and the python engine issue the same calls with a rheology ------------------------------------------
RHEO_CONFIGS = [c for c in ST.CONFIGS if c[4] == 0 and c[1] in (0, 1)]        # (the implicit flag is replaced by the rheology)
SPEC = dict(model="hb", k=0.02, n=1.0, tau_y=0.5, nu_max=2.0, beta=0.0, tol=1e-4, max_iter=7)


@pytest.fixture(scope="module")
def rheology_traces(tmp_path_factory):
    d = tmp_path_factory.mktemp("rheology_traces")
    stub = d / "sphk_stub.cpp"
    stub.write_text(ST.stub_source(os.path.join(ROOT, "include", "sphk.h")))
    exe = str(d / "rheology_trace_driver")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    cmd = [cxx, "-std=c++17", "-O0", "-I" + os.path.join(ROOT, "include"), "-I" + ST.HOST, "-I/usr/local/cuda/include", "-o", exe,
           os.path.join(ST.HOST, "sph_api.cpp"), str(stub), os.path.join(ROOT, "tests", "rheology_trace_driver.cpp"),
           "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe] + [ST.config_id(c) for c in RHEO_CONFIGS], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    traces = {}
    for line in r.stdout.splitlines():
        if line.startswith("TRACE "):
            _, key, *calls = line.split()
            traces[key] = calls
    assert sorted(traces) == sorted(ST.config_id(c) for c in RHEO_CONFIGS), r.stdout[-3000:]
    return traces


@pytest.mark.parametrize("config", RHEO_CONFIGS, ids=[ST.config_id(c) for c in RHEO_CONFIGS])
def test_layers_issue_the_same_calls_with_a_rheology(rheology_traces, config, monkeypatch):
    from cpp_fluid_particles_b200 import engine
    monkeypatch.setattr(engine.SphkOps, "rheology", SPEC)
    monkeypatch.setattr(ST, "NOT_COMPARED", ST.NOT_COMPARED | {"sphk_rheology_work_floats"})
    cpp = ST.compared(rheology_traces[ST.config_id(config)])
    py = ST.compared(ST.python_trace(config))
    assert "sphk_non_newtonian_viscosity" in cpp and "sphk_implicit_viscosity" not in cpp
    assert py == cpp
