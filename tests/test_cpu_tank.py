"""Tank motion without a device: the float64 schedule of tests/tank_ref.py against its own definition, sphk_tank_eval and
sphk_tank_accel_bound against it, every refusal of the host entries, the exported symbols and the python bindings, the headless app's
refusals, and the calls one step issues in the class layer and the python engine with a motion set.  numpy only."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import tank_ref as TR
import test_cpu_step_traces as ST
from util import ROOT

G = (0.0, -9.8, 0.0)
SPACE = (0.5, 0.3, 0.4)
ENTRIES = ("sphk_tank_eval", "sphk_tank_accel_bound", "sphk_tank_set", "sphk_tank_force", "sphk_tank_time", "sphk_tank_set_time")

MOTIONS = {
    "spin": dict(axis=(0.0, 2.0, 0.0), pivot=(0.25, 0.0, 0.2), spin=2.0, ramp=0.5),
    "roll": dict(axis=(0.0, 0.0, 1.0), pivot=(0.25, 0.0, 0.2), roll_amplitude=0.15, roll_omega=3.0, roll_phase=0.3, ramp=0.8),
    "harmonics": dict(accel=(0.5, 0.0, -0.25), harmonics=[dict(amplitude=(2.0, 0.0, 0.0), omega=6.0),
                                                          dict(amplitude=(0.0, 1.0, 0.5), omega=11.0, phase=0.7),
                                                          dict(amplitude=(-0.3, 0.2, 0.1), omega=2.5, phase=-1.0)], ramp=0.4),
    "no_ramp": dict(axis=(1.0, 0.0, 1.0), pivot=(0.1, 0.05, 0.3), roll_amplitude=-0.2, roll_omega=5.0, roll_phase=1.1, spin=0.7,
                    harmonics=[dict(amplitude=(1.0, 0.0, 0.0), omega=4.0)]),
}


def times(m):
    Tr = m.get("ramp", 0.0)
    if Tr == 0.0:
        return [0.0, 0.1, 1.0, 3.7]
    return [0.0, 0.3 * Tr, Tr - 1e-4, float(np.float32(Tr)), Tr + 1e-4, 2.0 * Tr, 3.7]


@pytest.fixture(scope="module")
def lib(pkg):
    from cpp_fluid_particles_b200 import capi
    return capi.sphk()


def fp(v):
    return (C.c_float * len(v))(*v)


def evaluate(lib, spec, t, g=G):
    from cpp_fluid_particles_b200 import capi
    out = (C.c_float * capi.TANK_STATE)()
    rc = lib.sphk_tank_eval(C.byref(capi.tank_motion(spec)), fp(g), C.c_double(t), out)
    return rc, np.array(out[:], np.float64)


@pytest.mark.parametrize("name", sorted(MOTIONS))
def test_reference_derivatives_match_the_angle(name):
    """tank_ref's thd and thdd are the derivatives of its theta (central differences away from the ramp's end), and theta_s is the
    integral of e Omega0"""
    m = MOTIONS[name]
    P = TR.params(m)
    h = 1e-5
    for t in [0.05, 0.31, 0.9, 1.7, 3.1]:
        if abs(t - P["Tr"]) < 3 * h:
            continue
        st = TR.state(m, G, t)
        d1 = (TR.theta(P, t + h) - TR.theta(P, t - h)) / (2 * h)
        d2 = (TR.theta(P, t + h) - 2 * TR.theta(P, t) + TR.theta(P, t - h)) / (h * h)
        assert abs(st[1] - d1) <= 1e-7 * max(1.0, abs(d1)), (t, st[1], d1)
        assert abs(st[2] - d2) <= 1e-3 * max(1.0, abs(d2)), (t, st[2], d2)
        s = np.linspace(0.0, t, 20001)
        e = np.minimum(1.0, s / P["Tr"]) if P["Tr"] > 0 else np.ones_like(s)
        assert abs(TR.spin_angle(P, t) - np.trapezoid(e * P["S"], s)) <= 1e-8 * max(1.0, abs(P["S"]) * t)


@pytest.mark.parametrize("name", sorted(MOTIONS))
def test_eval_matches_the_reference(lib, name):
    """sphk_tank_eval within 1e-6 relative of the float64 schedule before, at and after the ramp's end"""
    m = MOTIONS[name]
    ref = np.array([TR.state(m, G, t) for t in times(m)])
    got = np.array([evaluate(lib, m, t)[1] for t in times(m)])
    assert all(evaluate(lib, m, t)[0] == 0 for t in times(m))
    groups = [slice(0, 1), slice(1, 2), slice(2, 3), slice(3, 6), slice(6, 9)]
    for g in groups:
        scale = max(np.abs(ref[:, g]).max(), 1e-30)
        err = np.abs(got[:, g] - ref[:, g])
        assert np.all(err <= 1e-6 * np.abs(ref[:, g]) + 1e-7 * scale), (name, g, err.max(), scale)


def test_zero_motion_is_gravity(lib):
    """every amplitude zero: theta and its derivatives 0, R (G - a_w) = G exactly"""
    rc, s = evaluate(lib, dict(axis=(0.3, 0.4, 0.5), pivot=(0.1, 0.2, 0.3), ramp=0.5), 0.7)
    assert rc == 0
    assert np.array_equal(s, np.array([0, 0, 0, *np.float32(G), 0, 0, 0], np.float64))


@pytest.mark.parametrize("name", sorted(MOTIONS))
def test_accel_bound_covers_the_sampled_maximum(lib, name):
    from cpp_fluid_particles_b200 import capi
    m = MOTIONS[name]
    b = C.c_double(0.0)
    assert lib.sphk_tank_accel_bound(C.byref(capi.tank_motion(m)), fp(G), fp(SPACE), C.byref(b)) == 0
    assert np.isclose(b.value, TR.accel_bound(m, G, SPACE), rtol=1e-12)
    ts = np.linspace(0.0, 6.0, 6001)
    sampled = TR.sampled_accel(m, G, SPACE, ts)
    assert b.value >= sampled, (b.value, sampled)
    assert b.value <= 4.0 * sampled            # a bound, not a different quantity


BAD = [
    ("axis", dict(axis=(0.0, 0.0, 0.0))), ("axis_nan", dict(axis=(np.nan, 0.0, 1.0))), ("pivot_inf", dict(pivot=(np.inf, 0.0, 0.0))),
    ("amplitude_nan", dict(roll_amplitude=np.nan)), ("omega_negative", dict(roll_omega=-1.0)), ("phase_inf", dict(roll_phase=np.inf)),
    ("spin_nan", dict(spin=np.nan)), ("accel_inf", dict(accel=(0.0, -np.inf, 0.0))), ("ramp_negative", dict(ramp=-0.1)),
    ("ramp_nan", dict(ramp=np.nan)), ("harmonic_omega_negative", dict(harmonics=[dict(amplitude=(1.0, 0.0, 0.0), omega=-2.0)])),
    ("harmonic_amplitude_nan", dict(harmonics=[dict(amplitude=(np.nan, 0.0, 0.0), omega=2.0)])),
    ("harmonic_phase_inf", dict(harmonics=[dict(amplitude=(1.0, 0.0, 0.0), omega=2.0, phase=np.inf)])),
]


@pytest.mark.parametrize("name,spec", BAD, ids=[b[0] for b in BAD])
def test_host_entries_refuse(lib, name, spec):
    from cpp_fluid_particles_b200 import capi
    m = capi.tank_motion(spec)
    out, b = (C.c_float * capi.TANK_STATE)(), C.c_double(0.0)
    assert lib.sphk_tank_eval(C.byref(m), fp(G), C.c_double(0.1), out) == -1
    assert lib.sphk_tank_accel_bound(C.byref(m), fp(G), fp(SPACE), C.byref(b)) == -1


def test_host_entries_refuse_counts_times_and_pointers(lib):
    from cpp_fluid_particles_b200 import capi
    good = capi.tank_motion(MOTIONS["roll"])
    out, b = (C.c_float * capi.TANK_STATE)(), C.c_double(0.0)
    for n in (-1, capi.TANK_HARMONICS + 1):
        m = capi.tank_motion(MOTIONS["roll"])
        m.n_harmonics = n
        assert lib.sphk_tank_eval(C.byref(m), fp(G), C.c_double(0.1), out) == -1
    m = capi.tank_motion(MOTIONS["roll"])
    m.n_harmonics, m.harmonic_omega[3] = 3, -5.0       # entries past n_harmonics are ignored
    assert lib.sphk_tank_eval(C.byref(m), fp(G), C.c_double(0.1), out) == 0
    for t in (-1e-9, np.nan, np.inf):
        assert lib.sphk_tank_eval(C.byref(good), fp(G), C.c_double(t), out) == -1
    assert lib.sphk_tank_eval(C.byref(good), fp((0.0, np.nan, 0.0)), C.c_double(0.1), out) == -1
    assert lib.sphk_tank_eval(None, fp(G), C.c_double(0.1), out) == -1
    assert lib.sphk_tank_eval(C.byref(good), None, C.c_double(0.1), out) == -1
    assert lib.sphk_tank_eval(C.byref(good), fp(G), C.c_double(0.1), None) == -1
    for sp in ((0.0, 1.0, 1.0), (1.0, -1.0, 1.0), (1.0, np.nan, 1.0)):
        assert lib.sphk_tank_accel_bound(C.byref(good), fp(G), fp(sp), C.byref(b)) == -1
    assert lib.sphk_tank_accel_bound(C.byref(good), fp(G), fp(SPACE), None) == -1
    # the context entries refuse a NULL context before anything else
    assert lib.sphk_tank_set(None, C.byref(good), fp(G)) == -1
    assert lib.sphk_tank_force(None, None, C.c_float(0.001)) == -1
    assert lib.sphk_tank_time(None, C.byref(C.c_double()), None) == -1
    assert lib.sphk_tank_set_time(None, C.c_double(0.0)) == -1


def test_exports_header_and_capi(pkg):
    from cpp_fluid_particles_b200 import capi
    lib = os.path.join(ROOT, "cpp-fluid-particles_b200", "libsphk.so")
    if shutil.which("nm") is not None and os.path.exists(lib):
        syms = subprocess.run(["nm", "-D", lib], capture_output=True, text=True).stdout
        for name in ENTRIES:
            assert f" T {name}" in syms, name
    hdr = open(os.path.join(ROOT, "include", "sphk.h")).read()
    assert "#define SPHK_TANK_HARMONICS 4" in hdr and "#define SPHK_TANK_STATE 9" in hdr
    for name in ENTRIES:
        assert name in capi.SPHK_FUNCTIONS
    for name in ("sph_app_set_tank_motion", "sph_app_tank_state"):
        assert name in capi.SPH_APP_FUNCTIONS
    assert C.sizeof(capi.TankMotion) == 4 * (3 + 3 + 4 + 3 + 1 + 12 + 4 + 4 + 1)
    m = capi.tank_motion(MOTIONS["harmonics"])
    assert m.n_harmonics == 3 and list(m.harmonic_amplitude[1]) == [0.0, 1.0, 0.5] and m.harmonic_omega[3] == 0.0
    assert list(m.axis) == [0.0, 0.0, 1.0]
    with pytest.raises(ValueError):
        capi.tank_motion(dict(harmonics=[dict(omega=1.0)] * 5))
    with pytest.raises(ValueError):
        capi.tank_motion(dict(roll=1.0))
    with pytest.raises(ValueError):
        capi.tank_motion(dict(harmonics=[dict(frequency=1.0)]))


def test_python_refuses_bad_settings(lib):
    from cpp_fluid_particles_b200 import engine
    s = object.__new__(engine.SphkOps)
    s.L, s.ctx, s._G = lib, None, fp(G)
    for _, bad in BAD:
        with pytest.raises(ValueError):
            s.tank = bad
    assert s.tank is None
    s._thermal = dict(alpha=1e-4, beta=1e-3)
    with pytest.raises(ValueError):                          # heat transfer: the buoyancy acts along the constant G
        s.tank = MOTIONS["roll"]
    s._thermal, s.bodies_dynamic = None, True
    with pytest.raises(ValueError):                          # a rotating frame with dynamic bodies
        s.tank = MOTIONS["spin"]
    assert s.tank is None


@pytest.mark.parametrize("extra", [
    ["--tank-roll", "5"], ["--tank-roll", "5,1,0,0,0"], ["--tank-roll", "5,-1"], ["--tank-roll", "nan,1"], ["--tank-shake", "1,0,0"],
    ["--tank-shake", "1,0,0,-2"], ["--tank-accel", "1,0"], ["--tank-spin", "x"], ["--tank-spin", "1,2"], ["--tank-ramp", "-1"],
    ["--tank-roll", "5,1", "--ranks", "2"], ["--tank-roll", "5,1", "--heat", "1e-4,1e-3"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call"""
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


# ---- the class layer and the python engine issue the same calls with a motion set ----------------------------------------------
ROLL = dict(axis=(0.0, 0.0, 1.0), pivot=(0.25, 0.0, 0.25), roll_amplitude=0.1, roll_omega=4.0, ramp=0.5)
SHAKE = dict(harmonics=[dict(amplitude=(2.0, 0.0, 0.0), omega=6.0)])


@pytest.fixture(scope="module")
def tank_traces(tmp_path_factory):
    d = tmp_path_factory.mktemp("tank_traces")
    stub = d / "sphk_stub.cpp"
    stub.write_text(ST.stub_source(os.path.join(ROOT, "include", "sphk.h")))
    exe = str(d / "tank_trace_driver")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    cmd = [cxx, "-std=c++17", "-O0", "-I" + os.path.join(ROOT, "include"), "-I" + ST.HOST, "-I/usr/local/cuda/include", "-o", exe,
           os.path.join(ST.HOST, "sph_api.cpp"), str(stub), os.path.join(ROOT, "tests", "tank_trace_driver.cpp"),
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
def test_layers_issue_the_same_calls_with_a_tank_motion(tank_traces, config, monkeypatch):
    """sphk_tank_force where sphk_gravity was, once per step, in both layers; the rest of the step unchanged"""
    from cpp_fluid_particles_b200 import engine
    alloc = engine.SphkOps._alloc_solver_buffers

    def alloc_and_set(self, n):
        alloc(self, n)
        if config[5]:
            self.bodies_dynamic = True
        self.tank = SHAKE if config[5] else ROLL
    monkeypatch.setattr(engine.SphkOps, "_alloc_solver_buffers", alloc_and_set)
    cpp = ST.compared(tank_traces[ST.config_id(config)])
    py = ST.compared(ST.python_trace(config))
    assert cpp.count("sphk_tank_force") == 1 and "sphk_gravity" not in cpp
    assert py == cpp
