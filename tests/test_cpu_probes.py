"""Probes and water-level gauges without a device: the float64 reference (tests/probe_ref.py) on fields and profiles whose answer is
known, the exported symbols and header caps, the refusals of the python layers, the slab driver and the headless app, and the calls
one step issues in the class layer and the python engine with probes on.  numpy + scipy only."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import probe_ref as PR
import test_cpu_step_traces as ST
from util import ROOT

R, SPACING, M0 = 0.04, 0.02, 76.596750762082e-6


def _jittered_block(n=14, jitter=0.1, seed=5):
    rng = np.random.default_rng(seed)
    g = np.arange(n) * SPACING
    x = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    return x + rng.uniform(-jitter, jitter, x.shape) * SPACING


# ---- the reference's own checks ------------------------------------------------------------------------------------------------
def test_shepard_reproduces_a_constant_exactly():
    pos = _jittered_block()
    rng = np.random.default_rng(1)
    mass = M0 * rng.uniform(0.5, 2.0, len(pos))
    dens = rng.uniform(500.0, 1500.0, len(pos))
    vel = np.tile([0.3, -1.25, 2.0], (len(pos), 1))
    p = np.full(len(pos), 7.5)
    pts = rng.uniform(0.02, 0.24, (200, 3))
    v, m, _, _ = PR.records(pts, pos, vel, mass, dens, R, pressure=p, temperature=p)
    assert np.all(v[:, 7] > 0)
    assert np.allclose(v[:, 2:5], [0.3, -1.25, 2.0], rtol=1e-12, atol=0)
    assert np.allclose(v[:, 5:7], 7.5, rtol=1e-12, atol=0)
    # rho(x) = sum m W / sum V W: the particles' own density when it is uniform
    v2, _, _, _ = PR.records(pts, pos, vel, mass, np.full(len(pos), 1000.0), R)
    assert np.allclose(v2[:, 1], 1000.0, rtol=1e-12)
    assert np.isnan(v2[:, 5]).all() and np.isnan(v2[:, 6]).all()


def test_shepard_follows_a_linear_field_in_the_bulk():
    """first-order consistency is only approximate for Shepard on a jittered lattice: within a small part of a spacing's change"""
    pos = _jittered_block()
    grad = np.array([3.0, -2.0, 5.0])
    vel = np.tile(pos @ grad, (3, 1)).T
    rng = np.random.default_rng(2)
    pts = rng.uniform(0.08, 0.18, (300, 3))        # at least R from every face of the block
    v, _, _, _ = PR.records(pts, pos, vel, np.full(len(pos), M0), np.full(len(pos), 1000.0), R)
    err = np.abs(v[:, 2] - pts @ grad)
    assert err.max() <= 0.1 * SPACING * np.linalg.norm(grad), err.max()


def test_kernel_is_continuous_at_zero_and_at_R():
    assert PR.W(0.0, R) == 4.0 * PR.cW(R)
    assert PR.W(R, R) == 0.0 and PR.W(R * (1 + 1e-9), R) == 0.0
    assert abs(PR.W(1e-9, R) - PR.W(0.0, R)) < 1e-6 * PR.W(0.0, R)


def test_dry_points_and_dry_particles():
    pos = _jittered_block(4)
    v, m, lo, hi = PR.records([[5.0, 5.0, 5.0], [0.03, 0.03, 0.03]], pos, np.zeros_like(pos), np.full(len(pos), M0),
                              np.zeros(len(pos)), R)
    assert np.all(v[:, [0, 1, 2, 3, 4, 7]] == 0) and np.all(hi == 0)      # no particle has a volume
    v, _, _, _ = PR.records([[0.03, 0.03, 0.03]], pos, np.zeros_like(pos), np.full(len(pos), M0), np.full(len(pos), 1e3), R,
                            point_dry=np.array([True]))
    assert v[0, 7] == 0 and v[0, 0] == 0


@pytest.mark.parametrize("profile, want", [
    ([0.1, 0.2, 0.3, 0.2], -1.0),                            # dry
    ([0.9, 0.8, 0.7, 0.6], 3.0),                             # overtopped: |b - a|
    ([0.9, 0.7, 0.3, 0.1], 1.5),                             # the crossing half-way between samples 1 and 2
    ([0.9, 0.6, 0.2, 0.8, 0.1], 3.0 + 0.3 / 0.7),            # a droplet above the surface: the highest wet sample wins
    ([0.9, 0.5, 0.2, 0.1], 1.0),                             # theta met exactly at a sample
])
def test_gauge_crossings(profile, want):
    """hand-made S profiles with theta 0.5 on a gauge whose samples lie 1 apart"""
    level, bound, _ = PR.level_from_profile(np.array(profile), 0.5, float(len(profile) - 1))
    assert abs(level - want) <= 1e-12 + bound, (level, want)


def test_gauge_points_are_the_kernels_float_operations():
    pts = PR.gauge_points([0.1, 0.5, 0.2], [0.1, 0.0, 0.2], 7)
    assert pts.dtype == np.float32 and pts.shape == (7, 3)
    assert np.array_equal(pts[0], np.array([0.1, 0.5, 0.2], np.float32))
    assert np.array_equal(pts[-1], np.array([0.1, 0.0, 0.2], np.float32))


# ---- symbols, caps and refusals ----------------------------------------------------------------------------------------------
SPHK_NAMES = ("sphk_probe_sample", "sphk_probe_lattice", "sphk_gauge_levels", "sphk_probe_series_create", "sphk_probe_series_destroy",
              "sphk_probes_record", "sphk_probe_series_read")
APP_NAMES = ("sph_app_set_probes", "sph_app_probe_series", "sph_app_sample_probes", "sph_app_sample_lattice")


def test_exports(built):
    if shutil.which("nm") is None:
        pytest.skip("nm not available")
    d = os.path.join(ROOT, "cpp-fluid-particles_b200")
    k = subprocess.run(["nm", "-D", os.path.join(d, "libsphk.so")], capture_output=True, text=True).stdout
    h = subprocess.run(["nm", "-D", os.path.join(d, "libsphhost.so")], capture_output=True, text=True).stdout
    for name in SPHK_NAMES:
        assert f" T {name}" in k, name
    for name in APP_NAMES:
        assert f" T {name}" in h, name


def test_entries_without_a_device(built, pkg):
    """a series needs a device (SPHK_ERR_NO_DEVICE without one); the context entries refuse a NULL context before touching CUDA"""
    import torch
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    pts = np.zeros((1, 3), np.float32) + 0.1
    series = C.c_void_p()
    rc = L.sphk_probe_series_create(C.byref(series), pts.ctypes.data_as(C.c_void_p), C.c_int(1), None, C.c_int(0), C.c_float(0.5),
                                    C.c_int(4), None)
    if torch.cuda.is_available():
        assert rc == 0 and series.value
        L.sphk_probe_series_destroy(series)
    else:
        assert rc == -2 and not series.value                     # SPHK_ERR_NO_DEVICE
    out = np.zeros(8, np.float32)
    assert L.sphk_probe_sample(None, None, None, C.c_int(1), None, None, out.ctypes.data_as(C.c_void_p)) == -1
    assert L.sphk_gauge_levels(None, None, None, C.c_int(1), C.c_float(0.5), None) == -1
    assert L.sphk_probes_record(None, None, None, None, None) == -1
    # refused before any device work: too many points, a bad gauge, a zero capacity
    many = np.zeros((capi.PROBE_LIMIT + 1, 3), np.float32)
    assert L.sphk_probe_series_create(C.byref(series), many.ctypes.data_as(C.c_void_p), C.c_int(len(many)), None, C.c_int(0),
                                      C.c_float(0.5), C.c_int(4), None) == -1
    g, n = capi.gauge_structs([((0, 0.3, 0), (0, 0.0, 0), 8)], 0.5)
    g[0].samples = 1
    assert L.sphk_probe_series_create(C.byref(series), None, C.c_int(0), g, C.c_int(1), C.c_float(0.5), C.c_int(4), None) == -1
    assert L.sphk_probe_series_create(C.byref(series), pts.ctypes.data_as(C.c_void_p), C.c_int(1), None, C.c_int(0), C.c_float(0.5),
                                      C.c_int(0), None) == -1
    assert L.sphk_probe_series_create(C.byref(series), pts.ctypes.data_as(C.c_void_p), C.c_int(1), None, C.c_int(0), C.c_float(0.5),
                                      C.c_int(capi.PROBE_CAPACITY_LIMIT + 1), None) == -1


def test_header_caps_match_capi(pkg):
    from cpp_fluid_particles_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "sphk.h")).read()
    for name, value in (("SPHK_PROBE_FIELDS", capi.PROBE_FIELDS), ("SPHK_PROBE_LIMIT", capi.PROBE_LIMIT),
                        ("SPHK_GAUGE_LIMIT", capi.GAUGE_LIMIT), ("SPHK_GAUGE_MAX_SAMPLES", capi.GAUGE_MAX_SAMPLES),
                        ("SPHK_PROBE_CAPACITY_LIMIT", capi.PROBE_CAPACITY_LIMIT)):
        assert re.search(rf"#define {name} {value}\b", hdr), name
    assert C.sizeof(capi.SphkGauge) == 28
    for name in SPHK_NAMES:
        assert name in capi.SPHK_FUNCTIONS
    for name in APP_NAMES:
        assert name in capi.SPH_APP_FUNCTIONS


@pytest.mark.parametrize("points, gauges, threshold", [
    ([[0.1, float("nan"), 0.1]], [], 0.5),
    ([[0.1, 0.2]], [], 0.5),
    (np.zeros((4097, 3)), [], 0.5),
    ([], [((0.1, 0.2, 0.1), (0.1, 0.2, 0.1))], 0.5),                # a == b
    ([], [((0.1, 0.3, 0.1), (0.1, 0.0, 0.1), 1)], 0.5),             # k < 2
    ([], [((0.1, 0.3, 0.1), (0.1, 0.0, 0.1), 1025)], 0.5),
    ([], [((0.1, float("inf"), 0.1), (0.1, 0.0, 0.1))], 0.5),
    ([], [((0.1, 0.3, 0.1), (0.1, 0.0, 0.1))] * 65, 0.5),
    ([], [((0.1, 0.3, 0.1), (0.1, 0.0, 0.1))], 0.0),
    ([], [((0.1, 0.3, 0.1), (0.1, 0.0, 0.1))], float("nan")),
])
def test_python_refuses_bad_settings(pkg, points, gauges, threshold):
    from cpp_fluid_particles_b200 import capi, engine
    s = object.__new__(engine.SphkSystem)
    with pytest.raises(ValueError):
        s.set_probes(points, gauges, threshold)
    assert s._probe_series is None


def test_slabs_refuse_probes(pkg):
    from cpp_fluid_particles_b200 import slabs
    s = object.__new__(slabs.SlabSystem)
    with pytest.raises(ValueError):
        s.set_probes([[0.1, 0.1, 0.1]])


@pytest.mark.parametrize("extra", [
    ["--probe", "0.1,0.1", "--probe-out", "OUT"], ["--probe", "0.1,nan,0.1", "--probe-out", "OUT"],
    ["--probe", "x,0.1,0.1", "--probe-out", "OUT"], ["--probe", "0.1,0.1,0.1"],
    ["--gauge", "0.1,0.3,0.1,0.1,0.3,0.1", "--probe-out", "OUT"], ["--gauge", "0.1,0.3,0.1,0.1,0,0.1,1", "--probe-out", "OUT"],
    ["--gauge", "0.1,0.3,0.1,0.1,0,0.1,2.5", "--probe-out", "OUT"], ["--gauge", "0.1,0.3,0.1,0.1,0,0.1,1025", "--probe-out", "OUT"],
    ["--gauge", "0.1,0.3,0.1,0.1,0", "--probe-out", "OUT"],
    ["--gauge", "0.1,0.3,0.1,0.1,0,0.1", "--gauge-threshold", "0", "--probe-out", "OUT"],
    ["--gauge", "0.1,0.3,0.1,0.1,0,0.1", "--gauge-threshold", "inf", "--probe-out", "OUT"],
    ["--probe-out", "OUT"], ["--gauge-threshold", "0.5", "--probe", "0.1,0.1,0.1", "--probe-out", "OUT"],
    ["--probe", "0.1,0.1,0.1", "--probe-out", "OUT", "--ranks", "2"]])
def test_headless_refuses_bad_settings(built, extra, tmp_path):
    """refused while parsing, before any CUDA call (and nothing written)"""
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    out = tmp_path / "probes.csv"
    extra = [str(out) if a == "OUT" else a for a in extra]
    r = subprocess.run([cli, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr
    assert not out.exists()


def test_headless_refuses_too_many_probes(built, tmp_path):
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    args = []
    for _ in range(65):
        args += ["--gauge", "0.1,0.3,0.1,0.1,0,0.1"]
    r = subprocess.run([cli, "--frames", "0", "--probe-out", str(tmp_path / "z.csv")] + args, capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


# ---- the class layer and the python engine issue the same calls with probes on --------------------------------------------------
@pytest.fixture(scope="module")
def probe_traces(tmp_path_factory):
    d = tmp_path_factory.mktemp("probe_traces")
    stub = d / "sphk_stub.cpp"
    src = ST.stub_source(os.path.join(ROOT, "include", "sphk.h"))
    src = re.sub(r"int sphk_probe_series_create\(.*?\}\n", "", src, flags=re.S)    # the driver's (it hands out a series)
    stub.write_text(src)
    exe = str(d / "probe_trace_driver")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    cmd = [cxx, "-std=c++17", "-O0", "-I" + os.path.join(ROOT, "include"), "-I" + ST.HOST, "-I/usr/local/cuda/include", "-o", exe,
           os.path.join(ST.HOST, "sph_api.cpp"), str(stub), os.path.join(ROOT, "tests", "probe_trace_driver.cpp"),
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
def test_layers_record_at_the_same_place(probe_traces, class_layer_traces, config, monkeypatch):
    """one sphk_probes_record per step, the last call after the bodies' integration, in both layers; without it the step is the
    step without probes, call for call"""
    from cpp_fluid_particles_b200 import engine
    alloc = engine.SphkOps._alloc_solver_buffers

    def alloc_and_set(self, n):
        alloc(self, n)
        self._probe_series = C.c_void_p(1)
    monkeypatch.setattr(engine.SphkOps, "_alloc_solver_buffers", alloc_and_set)
    cpp = ST.compared(probe_traces[ST.config_id(config)])
    py = ST.compared(ST.python_trace(config))
    assert cpp.count("sphk_probes_record") == 1 and cpp[-1] == "sphk_probes_record"
    if config[5]:
        assert cpp[-2] == "sphk_bodies_integrate"
    assert py == cpp
    assert [c for c in cpp if c != "sphk_probes_record"] == ST.compared(class_layer_traces[ST.config_id(config)])


class_layer_traces = ST.class_layer_traces
