"""Open boundaries without a GPU: the library's host-only schedule and axes against tests/open_boundary_ref.py, the exported
symbols, argument validation of the device entries (NULL context), the refusals of the headless app and the slab driver, and
the scene sph_headless --emit-scene writes for --tap / --drain."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import open_boundary_ref as OB
from util import ROOT, bits

F = np.float32
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
INVALID = -1


def _lib():
    from cpp_fluid_particles_b200 import capi
    return capi.sphk(), capi


def _emitter(capi, **kw):
    e = {"origin": (0.3, 0.4, 0.2), "direction": (0.0, -1.0, 0.0), "speed": 1.0, "spacing": 0.02, "width": 4, "height": 3}
    e.update(kw)
    return e, capi.emitter_struct(e)


# ---- schedule ---------------------------------------------------------------------------------------------------------------
# u dt below, equal to and above s; the last case runs out of capacity mid-run
@pytest.mark.parametrize("speed,dt,spacing,cap_layers", [(1.3, 0.004, 0.02, None), (5.0, 0.004, 0.02, None),
                                                          (12.7, 0.004, 0.02, None), (7.9, 0.001, 0.005, 300)])
def test_schedule_matches_the_reference_over_1000_steps(built, speed, dt, spacing, cap_layers):
    L, capi = _lib()
    e, em = _emitter(capi, speed=speed, spacing=spacing)
    carry, ref_carry = C.c_double(0.0), 0.0
    used = refused = total = 0
    for step in range(1000):
        fit = 64 if cap_layers is None else min(64, cap_layers - used)
        off, sched = (C.c_float * 64)(), C.c_int(-1)
        assert L.sphk_emitter_advance(C.byref(em), C.byref(carry), C.c_float(dt), C.c_int(fit), off, C.byref(sched)) == 0
        ref_carry, k, ref_off = OB.advance(ref_carry, speed, spacing, dt, fit)
        assert sched.value == k and carry.value == ref_carry, step
        got = np.array(off[:min(k, fit)], F)
        assert np.array_equal(bits(got), bits(ref_off)), step
        assert (got >= 0).all() and (got < F(speed) * F(dt) + 1e-6).all()
        if k > 1:                                 # layers of one step lie exactly s apart along the stream
            assert np.allclose(np.diff(got.astype(np.float64)), -float(F(spacing)), rtol=0, atol=1e-6)
        used += min(k, fit)
        refused += k - min(k, fit)
        total += k
    # the schedule emits one layer per s of stream: the total is floor(1000 u dt / s), up to rounding of the sum
    assert abs(total - 1000 * float(F(speed)) * float(F(dt)) / float(F(spacing))) <= 1.0
    if cap_layers is not None:
        assert used == cap_layers and refused == total - cap_layers and refused > 0
    else:
        assert refused == 0


def test_schedule_validates_arguments(built):
    L, capi = _lib()
    e, em = _emitter(capi)
    carry, sched, off = C.c_double(0.0), C.c_int(0), (C.c_float * 4)()
    adv = lambda em=em, carry=carry, dt=0.004, mx=4, off=off, sched=C.byref(sched): L.sphk_emitter_advance(  # noqa: E731
        C.byref(em) if em is not None else None, C.byref(carry) if carry is not None else None, C.c_float(dt), C.c_int(mx), off, sched)
    assert adv() == 0
    assert adv(em=None) == INVALID and adv(carry=None) == INVALID and adv(sched=None) == INVALID
    assert adv(off=None) == INVALID and adv(off=None, mx=0) == 0 and adv(mx=-1) == INVALID
    for dt in (-0.001, float("nan"), float("inf")):
        assert adv(dt=dt) == INVALID
    assert adv(carry=C.c_double(-1.0)) == INVALID and adv(carry=C.c_double(float("nan"))) == INVALID
    assert adv(carry=C.c_double(0.02 * 70000)) == INVALID           # more than 65536 layers in one step
    for kw in ({"speed": 0.0}, {"speed": -1.0}, {"spacing": 0.0}, {"width": 0}, {"height": 0}, {"direction": (0, 0, 0)},
               {"origin": (float("nan"), 0, 0)}, {"speed": float("inf")}):
        _, bad = _emitter(capi, **kw)
        assert adv(em=bad) == INVALID, kw


# ---- axes -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", [(0, -1, 0), (0, 1, 0), (1, 0, 0), (0, 0, -1), (1, 2, 3), (0.3, -0.95, 0.1),
                                       (0.45, 0.9, 0.0), (0.43, 0.9, 0.0), (-2.0, 0.5, 7.0)])
def test_axes_match_the_reference(built, direction):
    L, capi = _lib()
    e, em = _emitter(capi, direction=direction)
    out = (C.c_float * 9)()
    assert L.sphk_emitter_axes(C.byref(em), out) == 0
    got = np.array(out[:], F).reshape(3, 3)
    ref = np.stack(OB.axes(**e))
    assert np.array_equal(bits(got), bits(ref))
    g = got.astype(np.float64)
    assert np.allclose(g @ g.T, np.eye(3), atol=1e-6)                      # orthonormal
    assert np.allclose(np.cross(g[1], g[0]), g[2], atol=1e-6)              # e2 = e1 x d
    d = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    assert np.allclose(g[0], d, atol=1e-7)
    # the rule: e1 is horizontal (d x y^) unless d is within about 25 degrees of vertical
    if abs(d[1]) > 0.9:
        assert abs(g[1, 0]) < 1e-7
    else:
        assert abs(g[1, 1]) < 1e-7


def test_axes_switch_at_0_9():
    """|d . y^| = 0.9 exactly (float32 direction) keeps d x y^; just above takes d x x^"""
    below = OB.axes((0, 0, 0), (np.sqrt(F(1) - F(0.81)), F(0.9), 0), 1, 1, 1, 1)
    above = OB.axes((0, 0, 0), (0.4, 0.92, 0.0), 1, 1, 1, 1)
    assert abs(float(below[1][1])) < 1e-7 and abs(float(above[1][0])) < 1e-7


# ---- exports and validation ---------------------------------------------------------------------------------------------------
def test_exported_symbols(built):
    from cpp_fluid_particles_b200 import capi
    L = C.CDLL(capi.LIBSPHK)
    for name in ("sphk_emitter_axes", "sphk_emitter_advance", "sphk_emit", "sphk_sinks_apply", "sphk_sinks_removed",
                 "sphk_fluid_set_count", "sphk_open_check"):
        assert hasattr(L, name), name
        assert name in capi.SPHK_FUNCTIONS
    H = C.CDLL(capi.LIBHOST, mode=C.RTLD_LOCAL)
    for name in ("sph_app_create_open", "sph_app_open_boundary_stats"):
        assert hasattr(H, name), name
        assert name in capi.SPH_APP_FUNCTIONS
    hdr = open(os.path.join(ROOT, "include", "sphk.h")).read()
    assert "#define SPHK_MAX_EMITTERS 16" in hdr and "#define SPHK_MAX_SINKS 16" in hdr
    assert C.sizeof(capi.SphkEmitter) == 40


def test_device_entries_validate_without_a_device(built):
    """NULL context and pointers are refused before any CUDA call"""
    L, capi = _lib()
    e, em = _emitter(capi)
    p = capi.SphkParticles()
    boxes = (C.c_float * 6)(0, 0, 0, 1, 1, 1)
    off = (C.c_float * 1)(0.0)
    out = C.c_int(0)
    assert L.sphk_emit(None, C.byref(p), 0, C.byref(em), 1, off, C.c_float(1e-4), C.c_float(0.004), None, 0) == INVALID
    assert L.sphk_sinks_apply(None, C.byref(p), boxes, 1) == INVALID
    assert L.sphk_sinks_removed(None, C.byref(out)) == INVALID
    assert L.sphk_fluid_set_count(None, None, 0) == INVALID
    assert L.sphk_open_check(None, C.byref(out)) == INVALID
    assert L.sphk_emitter_axes(None, (C.c_float * 9)()) == INVALID and L.sphk_emitter_axes(C.byref(em), None) == INVALID


# ---- refusals and the generated scene ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [["--tap", "1.0", "--ranks", "2"], ["--drain", "0.2", "--ranks", "2"], ["--tap", "-1"],
                                   ["--drain", "nan"], ["--capacity", "-5", "--tap", "1"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call"""
    r = subprocess.run([CLI, "--frames", "0"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 2, r.stderr


def test_headless_emit_scene_writes_the_emitter_and_sink(built, tmp_path, pkg):
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    prefix = str(tmp_path / "scene")
    r = subprocess.run([CLI, "--box", str(box), "--block", str(nx), str(ny), str(nz), "--origin", *[repr(float(o)) for o in origin],
                        "--tap", "2.5", "--drain", "0.2", "--emit-scene", prefix], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    e, sink = OB.tap_and_drain((box,) * 3, (nx, ny, nz), origin, 2.5, 0.2)
    got = np.fromfile(prefix + ".emitter.f32", F)
    want = np.array([*e["origin"], *e["direction"], e["speed"], e["spacing"], e["width"], e["height"]], F)
    assert np.array_equal(bits(got), bits(want))
    assert np.array_equal(bits(np.fromfile(prefix + ".sink.f32", F)), bits(sink))
    fluid = np.fromfile(prefix + ".fluid.f32", F).reshape(-1, 3)
    assert np.array_equal(bits(fluid), bits(pkg.scene.make_scene("mini").fluid))


def test_slab_system_refuses_open_boundaries(pkg):
    from cpp_fluid_particles_b200 import slabs
    sc = pkg.scene.make_scene("slabtest", "dfsph")
    with pytest.raises(ValueError):
        slabs.SlabSystem(sc, 0, 2, "cpu", sinks=[((0, 0, 0), (0.1, 0.1, 0.1))])
    with pytest.raises(ValueError):
        slabs.SlabSystem(sc, 0, 2, "cpu", emitters=[{"origin": (0.5, 0.5, 0.5), "direction": (0, -1, 0), "speed": 1.0,
                                                     "spacing": 0.02, "width": 2, "height": 2}])
