"""CFL-adaptive time stepping without a GPU: the library's host-only rule against tests/adaptive_dt_ref.py, the substep partition
of advance(), the exported symbols, argument validation of the device entries (NULL context), and the refusals of the headless
app and the slab driver."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import adaptive_dt_ref as AR
from util import ROOT, bits

F = np.float32
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
INVALID = -1
R = 0.04                       # the support radius of the reference scene (2 x spacing 0.02)
G = 9.8


def _lib():
    from cpp_fluid_particles_b200 import capi
    return capi.sphk(), capi


def _rule(capi, C_=0.2, dt_min=0.004 / 64, dt_max=0.004, radius=R, g=G):
    r = capi.SphkTimeStepRule()
    r.cfl, r.dt_min, r.dt_max, r.radius, r.gravity = C_, dt_min, dt_max, radius, g
    return r


def _step(L, r, v, dt_prev, remaining):
    dt, flags = C.c_float(-1.0), C.c_int(-1)
    rc = L.sphk_time_step(C.byref(r), C.c_double(v), C.c_double(dt_prev), C.c_double(remaining), C.byref(dt), C.byref(flags))
    return rc, F(dt.value), int(flags.value)


# ---- the rule -----------------------------------------------------------------------------------------------------------------
V = [0.0, 1e-9, 0.05, 0.5, 1.9, 2.0, 3.7, 12.0, 60.0, 1e3, 1e30, float("inf"), float("nan")]
PREV = [0.0, 0.004 / 64, 0.001, 0.004]
REMAIN = [0.0, -1.0, 1e-7, 0.004 / 128, 0.0012, 0.003, 0.0041, 0.0079, 0.008, 0.02]


@pytest.mark.parametrize("g", [0.0, G])
def test_rule_matches_the_reference_over_a_grid(built, g):
    """v = 0, non-finite, both clamps, the sliver case and remaining below dt_min, bit for bit with the same flags"""
    L, capi = _lib()
    r = _rule(capi, g=g)
    seen = 0
    for v in V:
        for dp in PREV:
            for rem in REMAIN:
                rc, dt, flags = _step(L, r, v, dp, rem)
                want, wflags = AR.rule(r.cfl, r.dt_min, r.dt_max, r.radius, r.gravity, v, dp, rem)
                assert rc == 0 and bits(np.array([dt])) == bits(np.array([want])) and flags == wflags, (v, dp, rem, dt, want, flags)
                seen |= flags
    assert seen == AR.MIN_CLAMP | AR.NONFINITE | AR.FRAME_END


def test_rule_cases(built):
    L, capi = _lib()
    r = _rule(capi)
    assert _step(L, r, 0.0, 0.0, 0.0) == (0, F(0.004), 0)                          # at rest: dt_max
    assert _step(L, r, 1.0, 0.0, 0.0) == (0, F(0.004), 0)                          # C R / v above dt_max
    assert _step(L, r, 4.0, 0.0, 0.0)[1] == F(0.2 * R / 4.0)                       # C R / v
    assert _step(L, r, 4.0, 0.004, 0.0)[1] == F(0.2 * R / (4.0 + G * 0.004))       # + |G| dt_prev
    assert _step(L, r, 1e4, 0.0, 0.0) == (0, F(0.004 / 64), AR.MIN_CLAMP)          # dt_min binds
    assert _step(L, r, float("nan"), 0.0, 0.0) == (0, F(0.004 / 64), AR.NONFINITE)
    assert _step(L, r, float("inf"), 0.0, 0.0) == (0, F(0.004 / 64), AR.NONFINITE)
    assert _step(L, r, 0.0, 0.0, 0.003) == (0, F(0.003), AR.FRAME_END)            # the frame ends with a shorter step
    assert _step(L, r, 0.0, 0.0, 0.006) == (0, F(0.003), 0)                        # no sliver: half of what is left
    assert _step(L, r, 0.0, 0.0, 0.008) == (0, F(0.004), 0)
    assert _step(L, r, 1e4, 0.0, 1e-6) == (0, F(1e-6), AR.MIN_CLAMP | AR.FRAME_END)  # the last substep may be below dt_min


def test_rule_validates_arguments(built):
    L, capi = _lib()
    dt, flags = C.c_float(), C.c_int()
    call = lambda r, v=1.0, dp=0.0, rem=0.0, d=C.byref(dt), f=C.byref(flags): L.sphk_time_step(  # noqa: E731
        C.byref(r) if r is not None else None, C.c_double(v), C.c_double(dp), C.c_double(rem), d, f)
    ok = _rule(capi)
    assert call(ok) == 0
    assert call(None) == INVALID and call(ok, d=None) == INVALID and call(ok, f=None) == INVALID
    nan, inf = float("nan"), float("inf")
    for kw in ({"C_": 0.0}, {"C_": -0.1}, {"C_": nan}, {"C_": inf}, {"dt_min": 0.0}, {"dt_min": 0.005}, {"dt_max": inf},
               {"dt_min": nan}, {"radius": 0.0}, {"radius": nan}, {"g": -1.0}, {"g": inf}):
        assert call(_rule(capi, **kw)) == INVALID, kw
    for kw in ({"v": -1.0}, {"dp": -1e-3}, {"dp": nan}, {"dp": inf}, {"rem": nan}, {"rem": inf}):
        assert call(ok, **kw) == INVALID, kw


# ---- the substep partition of advance() ------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_advance_partition_of_random_frames(built, seed):
    """the double sum of the float dts is within one float ulp of T, and the count is the rule's"""
    L, capi = _lib()
    rng = np.random.default_rng(seed)
    r = _rule(capi)
    for _ in range(40):
        T = float(rng.uniform(1e-5, 0.05))
        speeds = rng.uniform(0.0, 6.0, 400)
        start = dt_prev = float(F(rng.choice([0.0, 0.004, 0.0007])))
        elapsed, dts, end = 0.0, [], False
        while not end:
            rc, dt, flags = _step(L, r, speeds[len(dts)], dt_prev, T - elapsed)
            assert rc == 0
            end = bool(flags & AR.FRAME_END)
            dts.append(dt)
            elapsed += float(dt)
            dt_prev = float(dt)
        ref = AR.partition(T, lambda k: speeds[k], r.cfl, r.dt_min, r.dt_max, r.radius, r.gravity, start)
        assert np.array_equal(bits(np.array(dts, F)), bits(np.array(ref, F)))
        assert abs(math.fsum(float(d) for d in dts) - T) <= float(np.spacing(F(T))), T
        assert all(float(d) > 0 for d in dts)


def test_advance_partition_avoids_slivers(built):
    """at a constant bound, a frame of 2.5 dt_cfl ends with two equal steps of 0.75 dt_cfl, not with a sliver of 0.5"""
    L, capi = _lib()
    r = _rule(capi, g=0.0)
    dtc = float(F(0.2 * R / 4.0))
    got = AR.partition(2.5 * dtc, lambda k: 4.0, r.cfl, r.dt_min, r.dt_max, r.radius, 0.0, 0.0)
    assert len(got) == 3 and got[0] == F(dtc) and min(got) > 0.74 * dtc
    assert abs(float(got[1]) - float(got[2])) <= float(np.spacing(got[1]))
    elapsed, dts, end = 0.0, [], False
    while not end:
        rc, dt, flags = _step(L, r, 4.0, 0.0, 2.5 * dtc - elapsed)
        end = bool(flags & AR.FRAME_END)
        dts.append(dt)
        elapsed += float(dt)
    assert np.array_equal(bits(np.array(dts, F)), bits(np.array(got, F)))


# ---- exports and validation ---------------------------------------------------------------------------------------------------
def test_exported_symbols(built):
    from cpp_fluid_particles_b200 import capi
    L = C.CDLL(capi.LIBSPHK)
    for name in ("sphk_time_step", "sphk_step_speed", "sphk_step_speed_result"):
        assert hasattr(L, name), name
        assert name in capi.SPHK_FUNCTIONS
    H = C.CDLL(capi.LIBHOST, mode=C.RTLD_LOCAL)
    for name in ("sph_app_set_adaptive_dt", "sph_app_advance", "sph_app_adaptive_stats"):
        assert hasattr(H, name), name
        assert name in capi.SPH_APP_FUNCTIONS
    hdr = open(os.path.join(ROOT, "include", "sphk.h")).read()
    for flag in ("#define SPHK_DT_MIN_CLAMP 1", "#define SPHK_DT_NONFINITE 2", "#define SPHK_DT_FRAME_END 4"):
        assert flag in hdr
    assert C.sizeof(capi.SphkTimeStepRule) == 40


def test_device_entries_validate_without_a_device(built):
    """NULL context and pointers are refused before any CUDA call"""
    L, capi = _lib()
    p = capi.SphkParticles()
    v, bad = (C.c_float * 2)(), C.c_int(0)
    assert L.sphk_step_speed(None, C.byref(p), 0) == INVALID
    assert L.sphk_step_speed(None, None, 1) == INVALID
    assert L.sphk_step_speed_result(None, v, C.byref(bad)) == INVALID


# ---- refusals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [["--cfl", "0.2", "--ranks", "2"], ["--cfl", "-0.2"], ["--cfl", "nan"], ["--cfl", "0.2", "--dt-min", "inf"],
                                   ["--cfl", "0.2", "--dt-min", "-1"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call"""
    r = subprocess.run([CLI, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


def test_slab_system_refuses_adaptive_time_stepping(pkg):
    from cpp_fluid_particles_b200 import slabs
    sc = pkg.scene.make_scene("slabtest", "dfsph")
    with pytest.raises(ValueError):
        slabs.SlabSystem(sc, 0, 2, "cpu", adaptive={"C": 0.2})
