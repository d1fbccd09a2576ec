"""Open boundaries on the GPU: closed systems unchanged, removal plus emission equal to a rebuilt closed system bit for bit on
every execution path, emission and sink classification per element against tests/open_boundary_ref.py, the count bookkeeping,
a ballistic jet and a draining tank, the layers (facade, python engine, sph_headless) agreeing bit for bit, validation and
refusals, and sph_headless --tap --drain with blocking launches."""
import ctypes as C
import dataclasses
import os
import shutil
import subprocess

import numpy as np
import pytest

import open_boundary_ref as OB
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
INVALID, CAPACITY, STATE = -1, -3, -4


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _np(t):
    return t.detach().cpu().numpy().copy()


def _same(a, b, what, n=None):
    for f in ("pos", "vel", "density", "pressure"):
        x, y = np.asarray(a[f]), np.asarray(b[f])
        if n is not None:
            x, y = x[:n], y[:n]
        assert x.shape == y.shape and np.array_equal(bits(x), bits(y)), f"{what}: {f} differs"


def _box(sc, lo, hi):
    return (tuple(float(F(x)) for x in lo), tuple(float(F(x)) for x in hi))


# ---- 1. closed systems are unchanged ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_closed_system_is_unchanged(pkg, built, solver):
    """the open constructors without emitters and sinks, with capacity n and 2n: same bits, launches and step graph"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", solver)
    n = sc.fluid.shape[0]
    old = capi.SphApp(sc)
    new = [capi.SphApp(sc, max_fluid=cap, emitters=[], sinks=[]) for cap in (n, 2 * n)]
    for _ in range(4):
        old.step()
        for a in new:
            a.step()
    ref = old.download()
    for a in new:
        _same(a.download(), ref, f"{solver}: facade")
        assert a.step_graph_active() == old.step_graph_active()
        assert a.open_boundary_stats() == ({"emitted": 0, "removed": 0, "refused": 0}, 0)
    for a in [old] + new:
        a.close()
    s0 = engine.SphkSystem(sc)
    ss = [engine.SphkSystem(sc, max_fluid=cap, emitters=[], sinks=[]) for cap in (n, 2 * n)]
    for _ in range(3):
        s0.step()
        for s in ss:
            s.step()
    st = s0.state()
    for s in ss:
        assert not s.open
        _same(s.state(), st, f"{solver}: engine")
        assert s.launch_count() == s0.launch_count()
        s.close()
    s0.close()


# ---- 2. removal and emission equal a rebuilt closed system ------------------------------------------------------------------
def _open_scene(pkg, solver, adaptive=False):
    if solver == "dfsph" and adaptive:
        sc = pkg.scene.make_scene("mini", "dfsph", dt=0.004)
    else:
        sc = pkg.scene.benchmark_scene("mini", solver)
    dt = float(sc.params.dt)
    lo = sc.fluid.min(0)
    # a jet into the box beside the block, whose layers reach the second sink; the first sink takes a corner of the block
    em = {"origin": (0.06, 0.40, 0.40), "direction": (1.0, -0.2, 0.1), "speed": 0.02 / dt * 1.7, "spacing": 0.02, "width": 3,
          "height": 2}
    sinks = [_box(sc, lo - 0.001, lo + np.array([0.05, 0.03, 0.05], F)), ((0.10, 0.30, 0.36), (0.20, 0.45, 0.45))]
    return sc, em, sinks


@pytest.mark.parametrize("path", ["list", "tile", "cells"])
@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "dfsph_adaptive", "pbd"])
def test_removal_and_emission_equal_a_rebuilt_system(pkg, built, solver, path):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    base = solver.split("_")[0]
    sc, em, sinks = _open_scene(pkg, base, adaptive=solver.endswith("adaptive"))
    n0 = sc.fluid.shape[0]
    cap = n0 + 600
    use_list = path != "cells"
    s = engine.SphkSystem(sc, step0=False, max_fluid=cap, emitters=[em], sinks=sinks, use_list=use_list)
    if path == "tile":
        s.set_option(capi.OPT_TILE, 1)
    if base == "pbd":
        s.step()                                  # the first PBD step only initialises the last positions (Q6)
    boxes = capi.sink_boxes(sinks)
    seen_removed = seen_emitted = 0
    for k in range(4):
        n = s.fluid.n
        pre = {f: _np(getattr(s.fluid, f)[:n]) for f in ("pos", "vel", "density", "pressure")}
        dens_slots, pres_slots = _np(s.fluid.density), _np(s.fluid.pressure)
        h, kind = s._history()
        hist = _np(h[:n]) if h is not None else None
        carry = s.emitter_carry[0]
        st0 = s.open_boundary_stats()
        s.step()
        st1 = s.open_boundary_stats()
        removed, emitted = st1["removed"] - st0["removed"], st1["emitted"] - st0["emitted"]
        L = s.fluid.n
        assert L == n + emitted - removed
        # the rebuilt closed system: survivors, then the emitted particles, in that order
        keep = ~OB.sink_mask(pre["pos"], boxes)
        assert int((~keep).sum()) == removed
        _, layers, offs = OB.advance(carry, em["speed"], em["spacing"], sc.params.dt, 1 << 20)
        epos, evel = OB.layers(em, offs)
        assert epos.shape[0] == emitted
        pos = np.concatenate([pre["pos"][keep], epos], 0)
        vel = np.concatenate([pre["vel"][keep], np.repeat(evel[None, :], emitted, 0)], 0)
        r = engine.SphkSystem(dataclasses.replace(sc, fluid=np.ascontiguousarray(pos)), step0=False, max_fluid=cap, use_list=use_list)
        if path == "tile":
            r.set_option(capi.OPT_TILE, 1)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(r.device)  # noqa: E731
        r.fluid.pos[:L] = dev(pos)
        r.fluid.vel[:L] = dev(vel)
        r.fluid.density[:L] = dev(dens_slots[:L])         # density and pressure stay in their slots (Q2)
        r.fluid.pressure[:L] = dev(pres_slots[:L])
        rh, _ = r._history()
        if kind == 1:
            rh[:L] = dev(np.concatenate([hist[keep], np.zeros(emitted, F)]))
        elif kind == 2:
            rh[:L] = dev(np.concatenate([hist[keep], epos - F(sc.params.dt) * evel[None, :]], 0))
            r.pos_last_init = True
        r.emitter_carry = []
        r.step()
        a, b = s.state(), r.state()
        _same(a, b, f"{solver}/{path} step {k}", L)
        assert np.array_equal(_np(s.cs_fluid), _np(r.cs_fluid)), "cell_start"
        if h is not None:
            assert np.array_equal(bits(_np(h[:L])), bits(_np(rh[:L]))), "history"
        if base == "dfsph":
            assert (s.it_div, s.it_den) == (r.it_div, r.it_den)
        assert s.open_check() == 0
        r.close()
        seen_removed += removed
        seen_emitted += emitted
    assert seen_removed > 0 and seen_emitted > 0
    s.close()


# ---- 3. emission per element -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["one", "several", "w1h1", "oblique", "refused"])
def test_emission_per_element(pkg, built, case):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    solver = {"one": "dfsph", "several": "pbd", "w1h1": "wcsph", "oblique": "pbd", "refused": "dfsph"}[case]
    sc = pkg.scene.benchmark_scene("mini", solver)
    dt = float(sc.params.dt)
    n = sc.fluid.shape[0]
    em = {"origin": (0.25, 0.40, 0.25), "direction": (0.0, -1.0, 0.0), "speed": 1.0, "spacing": 0.02, "width": 5, "height": 4}
    speed = {"one": 0.025 / dt, "several": 0.07 / dt, "w1h1": 0.05 / dt, "oblique": 0.03 / dt, "refused": 0.07 / dt}[case]
    em["speed"] = speed
    if case == "w1h1":
        em.update(width=1, height=1)
    if case == "oblique":
        em.update(direction=(0.3, -0.8, 0.5), width=3, height=6)
    per = em["width"] * em["height"]
    cap = n + per + 7 if case == "refused" else n + 400
    s = engine.SphkSystem(sc, step0=False, max_fluid=cap, emitters=[em])
    h, kind = s._history()
    if h is not None:
        h.fill_(123.0)
    s.fluid.pos[n:] = 77.0
    before = {f: _np(getattr(s.fluid, f)) for f in ("pos", "vel", "mass")}
    e = s.open_emit()
    s.synchronize()
    _, k, offs = OB.advance(0.0, em["speed"], em["spacing"], dt, (cap - n) // per)
    assert {"one": 1, "several": 3, "w1h1": 2, "oblique": 1, "refused": 3}[case] == k
    pos, vel = OB.layers(em, offs)
    assert e == pos.shape[0] == min(k, (cap - n) // per) * per
    got = _np(s.fluid.pos)
    assert np.array_equal(bits(got[n:n + e]), bits(pos)), "positions"
    assert np.array_equal(bits(_np(s.fluid.vel)[n:n + e]), bits(np.repeat(vel[None, :], e, 0))), "velocities"
    d = OB.axes(**em)[0]
    assert np.array_equal(bits(vel), bits((F(em["speed"]) * d).astype(F)))
    assert (_np(s.fluid.mass)[n:n + e] == F(sc.params.m0)).all()
    assert (_np(s.fluid.density)[n:n + e] == 0).all() and (_np(s.fluid.pressure)[n:n + e] == 0).all()
    if kind == 1:
        assert (_np(h)[n:n + e] == 0).all()
    elif kind == 2:
        assert np.array_equal(bits(_np(h)[n:n + e]), bits((pos - F(dt) * vel[None, :]).astype(F)))
    if h is not None:
        assert (_np(h)[n + e:] == 123.0).all()
    # slots beyond the emitted ones are untouched
    for f in ("pos", "vel", "mass"):
        assert np.array_equal(bits(_np(getattr(s.fluid, f))[n + e:]), bits(before[f][n + e:])), f
    st = s.open_boundary_stats()
    assert st["emitted"] == e and st["refused"] == (k * per - e)
    if case == "refused":
        assert st["refused"] == 2 * per
    s.close()


# ---- 4. sink classification -----------------------------------------------------------------------------------------------
def test_sink_classification(pkg, built):
    """lo is inside, hi is outside, on every axis; the count equals numpy's on the positions before the step"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    lo, hi = np.array([0.15, 0.07, 0.15], F), np.array([0.23, 0.15, 0.21], F)
    s = engine.SphkSystem(sc, step0=False, sinks=[(lo, hi)])
    pos = _np(s.fluid.pos)
    probes = [lo, hi, [lo[0], lo[1], hi[2]], [hi[0], lo[1], lo[2]], [lo[0], hi[1], lo[2]],
              np.nextafter(hi, np.float32(0)), np.nextafter(lo, np.float32(0))]
    for i, p in enumerate(probes):
        pos[i] = np.asarray(p, F)
    s.fluid.pos[: pos.shape[0]] = torch.from_numpy(pos).to(s.device)
    s.fluid.vel.fill_(0.5)
    want = OB.sink_mask(pos, capi.sink_boxes([(lo, hi)]))
    assert list(want[:7]) == [True, False, False, False, False, True, False]
    p = s.fluid.abi()
    boxes = capi.sink_boxes([(lo, hi)])
    fp = boxes.ctypes.data_as(C.POINTER(C.c_float))
    assert s.L.sphk_sinks_apply(s.ctx, C.byref(p), fp, 1) == 0
    removed = C.c_int(-1)
    assert s.L.sphk_sinks_removed(s.ctx, C.byref(removed)) == 0
    assert removed.value == int(want.sum()) > 10
    got, v = _np(s.fluid.pos), _np(s.fluid.vel)
    assert (got[want] == F(-1e6)).all() and (v[want] == 0).all()
    assert np.array_equal(bits(got[~want]), bits(pos[~want])) and (v[~want] == F(0.5)).all()
    s.close()


# ---- 5. bookkeeping ---------------------------------------------------------------------------------------------------------
def _tap_app(pkg, solver, tap=1.5, drain=0.2, capacity=None):
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", solver)
    box, block, origin = pkg.scene._CONFIGS["mini"]
    e, sink = OB.tap_and_drain((box,) * 3, block, origin, tap, drain)
    sinks = [(sink[:3], sink[3:])] if drain > 0 else []
    n = sc.fluid.shape[0]
    return capi.SphApp(sc, max_fluid=capacity or 2 * n, emitters=[e], sinks=sinks), n


def test_bookkeeping_over_200_frames(pkg, built):
    _gpu()
    app, n0 = _tap_app(pkg, "dfsph", tap=2.0, drain=0.25)
    for k in range(200):
        app.step()
        st, check = app.open_boundary_stats()
        assert app.fluid_count == n0 + st["emitted"] - st["removed"], k
        assert check == 0, k
    assert st["emitted"] > 0 and st["removed"] > 0
    d = app.download()
    assert d["pos"].shape[0] == app.fluid_count and np.isfinite(d["pos"]).all()
    # a live particle moved outside the grid by a host-side edit: the count check reports it
    d["pos"][0] = (-0.3, -0.3, -0.3)
    app.upload(pos=d["pos"])
    app.step()
    assert app.open_boundary_stats()[1] == 1
    app.close()


def test_without_a_drain_the_count_grows_to_capacity(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "pbd")
    n0 = sc.fluid.shape[0]
    box, block, origin = pkg.scene._CONFIGS["mini"]
    e, _ = OB.tap_and_drain((box,) * 3, block, origin, 5.0, 0.0)
    cap = n0 + 64 * 12 + 5
    app = capi.SphApp(sc, max_fluid=cap, emitters=[e], sinks=[])
    counts = []
    for _ in range(60):
        app.step()
        counts.append(app.fluid_count)
    st, check = app.open_boundary_stats()
    assert all(b >= a for a, b in zip(counts, counts[1:])) and counts[-1] == n0 + 64 * 12
    assert st["refused"] > 0 and st["refused"] % 64 == 0 and st["removed"] == 0 and check == 0
    app.close()


# ---- 6. physics -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_horizontal_jet_is_ballistic(pkg, built, solver):
    """one particle per layer, layers 0.05 apart (beyond the support radius): the first layer follows o + u t + g t^2 / 2 within
    2 % of the distance travelled for 20 steps"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", solver)
    dt = float(sc.params.dt)
    em = {"origin": (0.05, 0.42, 0.42), "direction": (1.0, 0.0, 0.0), "speed": 3.0, "spacing": 0.05, "width": 1, "height": 1}
    app = capi.SphApp(sc, max_fluid=sc.fluid.shape[0] + 100, emitters=[em], sinks=[])
    carry, steps, delta = 0.0, 0, None       # the constructor's step 0 runs the schedule once
    carry, k, offs = OB.advance(carry, 3.0, 0.05, dt, 100)
    if k:
        delta, steps = float(offs[0]), 1
    while delta is None:
        app.step()
        carry, k, offs = OB.advance(carry, 3.0, 0.05, dt, 100)
        if k:
            delta, steps = float(offs[0]), 1
    o = np.array(em["origin"], np.float64)
    worst = 0.0
    for _ in range(20):
        app.step()
        steps += 1
        p = app.download()["pos"].astype(np.float64)
        jet = p[(p[:, 2] > 0.39) & (p[:, 1] > 0.3)]
        first = jet[np.argmax(jet[:, 0])]
        t = steps * dt
        want = o + np.array([delta + 3.0 * t, -0.5 * 9.8 * t * t, 0.0])
        travelled = np.linalg.norm(want - o)
        worst = max(worst, float(np.linalg.norm(first - want) / travelled))
    print(f"\n{solver}: worst deviation of the first layer from o + u t + g t^2/2: {worst:.4f} of the distance travelled")
    assert worst <= 0.02
    app.close()


def test_draining_tank_only_loses_particles_inside_the_drain(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    drain = np.array([0.0, 0.0, 0.0, 0.22, 0.03, 0.22], F)
    app = capi.SphApp(sc, max_fluid=sc.fluid.shape[0], emitters=[], sinks=[(drain[:3], drain[3:])])
    prev = app.open_boundary_stats()[0]["removed"]
    count = app.fluid_count
    total = 0
    for _ in range(60):
        pos = app.download()["pos"]
        inside = int(OB.sink_mask(pos, drain).sum())
        app.step()
        st = app.open_boundary_stats()[0]
        assert st["removed"] - prev == inside
        assert app.fluid_count == count - inside
        prev, count, total = st["removed"], app.fluid_count, total + inside
    assert total > 0
    app.close()


# ---- 7. the layers agree ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [[], ["--stir", "6"], ["--implicit-viscosity", "0.05"]])
def test_layers_agree(pkg, built, tmp_path, extra):
    """sph_headless --tap --drain, the python engine and (without --stir, which it cannot combine) the facade: same bits after
    6 frames"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    prefix = str(tmp_path / "s")
    base = [CLI, "--solver", "dfsph", "--iters", "4", "--box", str(box), "--block", str(nx), str(ny), str(nz), "--origin",
            *[repr(float(o)) for o in origin], "--tap", "2.0", "--drain", "0.25"] + extra
    r = subprocess.run(base + ["--emit-scene", prefix], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    ev = np.fromfile(prefix + ".emitter.f32", F)
    em = {"origin": ev[:3], "direction": ev[3:6], "speed": ev[6], "spacing": ev[7], "width": int(ev[8]), "height": int(ev[9])}
    sk = np.fromfile(prefix + ".sink.f32", F)
    fluid = np.fromfile(prefix + ".fluid.f32", F).reshape(-1, 3)
    sc = dataclasses.replace(pkg.scene.benchmark_scene("mini", "dfsph"), fluid=fluid)
    cap = 2 * fluid.shape[0]
    bodies = None
    if "--stir" in extra:
        bs = np.fromfile(prefix + ".body_state.f32", F)
        bodies = [{"points": np.fromfile(prefix + ".body.f32", F).reshape(-1, 3), "position": bs[:3], "orientation": bs[3:7],
                   "linear_velocity": bs[7:10], "angular_velocity": bs[10:13]}]
    s = engine.SphkSystem(sc, max_fluid=cap, emitters=[em], sinks=[(sk[:3], sk[3:])], bodies=bodies)
    app = None if bodies else capi.SphApp(sc, max_fluid=cap, emitters=[em], sinks=[(sk[:3], sk[3:])])
    if "--implicit-viscosity" in extra:
        s.implicit_nu = s.implicit_nu_boundary = 0.05
        app.set_implicit_viscosity(0.05, 0.05)
    frames = 6
    for _ in range(frames):
        s.step()
        if app:
            app.step()
    st = s.state()
    if app:
        _same(app.download(), st, "facade vs engine")
        assert app.open_boundary_stats()[0] == s.open_boundary_stats()
        app.close()
    r = subprocess.run(base + ["--frames", str(frames), "--quiet", "--dump", prefix], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    pos = np.fromfile(prefix + ".pos.f32", F).reshape(-1, 3)
    den = np.fromfile(prefix + ".density.f32", F)
    assert np.array_equal(bits(pos), bits(st["pos"])) and np.array_equal(bits(den), bits(st["density"])), "sph_headless"
    import json
    summary = json.loads(r.stdout.strip().splitlines()[-1])
    o = s.open_boundary_stats()
    assert (summary["fluid_count"], summary["emitted"], summary["removed"], summary["refused"]) == \
        (s.fluid_count, o["emitted"], o["removed"], o["refused"])
    assert o["emitted"] > 0
    s.close()


# ---- 8. validation and refusals ---------------------------------------------------------------------------------------------
def test_entries_validate_arguments(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    from cpp_fluid_particles_b200.engine import _ptr
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    n = sc.fluid.shape[0]
    s = engine.SphkSystem(sc, step0=False, max_fluid=n + 100)
    L, ctx = s.L, s.ctx
    em = capi.emitter_struct({"origin": (0.25, 0.4, 0.25), "direction": (0, -1, 0), "speed": 1.0, "spacing": 0.02,
                                       "width": 5, "height": 4})
    p = s.fluid.abi()
    off = (C.c_float * 8)(0.0, 0.01, 0.02, 0.0, 0.0, 0.0, 0.0, 0.0)
    f, i = C.c_float, C.c_int

    def emit(dst=n, layers=1, offs=off, m0=1e-4, dt=0.004, hist=None, kind=0, emitter=em, part=p):
        return L.sphk_emit(ctx, C.byref(part) if part is not None else None, i(dst), C.byref(emitter), i(layers), offs, f(m0), f(dt),
                           hist, i(kind))

    assert emit(part=None) == INVALID and emit(layers=-1) == INVALID and emit(dst=-1) == INVALID and emit(offs=None) == INVALID
    assert emit(m0=0.0) == INVALID and emit(dt=-1.0) == INVALID and emit(kind=3) == INVALID and emit(kind=1) == INVALID
    bad = (C.c_float * 1)(float("nan"))
    assert emit(offs=bad) == INVALID
    assert emit(layers=6) == CAPACITY and emit(dst=n + 81) == CAPACITY
    boxes = capi.sink_boxes([((0.1, 0.1, 0.1), (0.2, 0.2, 0.2))])
    fb = lambda b: np.ascontiguousarray(b, F).ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    for b in ([[0.2, 0.1, 0.1, 0.1, 0.2, 0.2]], [[0.1, 0.1, 0.1, 0.1, 0.2, 0.2]], [[float("nan"), 0, 0, 1, 1, 1]]):
        assert L.sphk_sinks_apply(ctx, C.byref(p), fb(b), 1) == INVALID
    assert L.sphk_sinks_apply(ctx, C.byref(p), fb(np.zeros((17, 6))), 17) == INVALID
    assert L.sphk_sinks_apply(ctx, C.byref(p), fb(boxes), -1) == INVALID
    r = C.c_int(0)
    assert L.sphk_sinks_removed(ctx, C.byref(r)) == STATE          # before the first sphk_sinks_apply
    # set_count: after a search only, before the first sweep, L <= the searched count
    s.search_fluid()
    assert L.sphk_fluid_set_count(ctx, _ptr(s.cs_fluid), i(n + 1)) == STATE
    assert L.sphk_fluid_set_count(ctx, _ptr(s.cs_fluid), i(-1)) == INVALID
    assert L.sphk_fluid_set_count(ctx, None, i(n)) == INVALID
    assert L.sphk_fluid_set_count(ctx, _ptr(s.cs_fluid), i(n)) == 0
    s.density()
    assert L.sphk_fluid_set_count(ctx, _ptr(s.cs_fluid), i(n)) == STATE      # after a sweep
    assert emit() == 0
    assert L.sphk_density(ctx, s._s()) == STATE                              # the emitted slots need a search first
    s.search_fluid()
    # active range (slab ranks)
    L.sphk_set_active_range(ctx, i(0), i(n // 2))
    assert emit() == STATE and L.sphk_sinks_apply(ctx, C.byref(p), fb(boxes), 1) == STATE
    assert L.sphk_fluid_set_count(ctx, _ptr(s.cs_fluid), i(n)) == STATE
    L.sphk_set_active_range(ctx, i(0), i(-1))
    assert L.sphk_sinks_apply(ctx, C.byref(p), fb(boxes), 1) == 0 and L.sphk_sinks_removed(ctx, C.byref(r)) == 0
    s.close()
    with pytest.raises(ValueError):
        engine.SphkSystem(sc, step0=False, sinks=[((0.2, 0.1, 0.1), (0.1, 0.2, 0.2))])
    with pytest.raises(RuntimeError):
        engine.SphkSystem(sc, step0=False, emitters=[{"origin": (0.2, 0.2, 0.2), "direction": (0, 0, 0), "speed": 1.0, "spacing": 0.02}])


def test_facade_refusals(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    n = sc.fluid.shape[0]
    good = {"origin": (0.25, 0.4, 0.25), "direction": (0, -1, 0), "speed": 1.0, "spacing": 0.02, "width": 4, "height": 4}
    for bad_e, bad_s, cap in ((dict(good, origin=(0.01, 0.4, 0.25)), [], 2 * n),        # layer outside the clamp box
                              (dict(good, origin=(0.25, 0.4944, 0.25), direction=(0, 1, 0)), [], 2 * n),   # advanced layer outside
                              (dict(good, speed=-1.0), [], 2 * n), (dict(good, width=0), [], 2 * n),
                              (good, [((0.2, 0.1, 0.1), (0.1, 0.2, 0.2))], 2 * n), (good, [], n - 1)):
        with pytest.raises(RuntimeError):
            capi.SphApp(sc, max_fluid=cap, emitters=[bad_e], sinks=bad_s)
    with pytest.raises(RuntimeError):
        capi.SphApp(sc, max_fluid=2 * n, emitters=[good] * 17, sinks=[])
    app = capi.SphApp(sc, max_fluid=2 * n, emitters=[good], sinks=[])
    a = np.zeros((n, 3), F)
    with pytest.raises(RuntimeError):
        app.submit(a, a)                      # the pipelined path assumes a fixed count
    assert not app.step_graph_active()
    for _ in range(4):
        app.step()
    assert not app.step_graph_active()       # open systems never capture a step graph
    app.close()


CLASS_REFUSALS = r"""
#include <cstdio>
#include <memory>
#include "sph_api.hpp"
struct Other : BaseSolver {
    void step(std::shared_ptr<SPHParticles>&, const std::shared_ptr<SPHParticles>&, const DArray<int>&, const DArray<int>&, float3,
              int3, float, float, float, float, float, float, float, float3, float, float) override {}
protected:
    void advect(std::shared_ptr<SPHParticles>&, float, float3) override {}
    void force(std::shared_ptr<SPHParticles>&, float, float3) override {}
};
int main() {
    std::vector<float3> f, b;
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) for (int k = 0; k < 6; ++k)
        f.push_back(make_float3(0.15f + 0.02f * i, 0.1f + 0.02f * j, 0.15f + 0.02f * k));
    for (int i = 0; i < 20; ++i) for (int k = 0; k < 20; ++k) b.push_back(make_float3(0.02f + 0.0235f * i, 0.005f, 0.02f + 0.0235f * k));
    sphb200::OpenBoundaries ob;
    ob.sinks.push_back({make_float3(0.0f, 0.0f, 0.0f), make_float3(0.1f, 0.05f, 0.1f)});
    const float3 space = make_float3(0.5f, 0.5f, 0.5f), G = make_float3(0.0f, -9.8f, 0.0f);
    const int3 cells = make_int3(13, 13, 13);
    int active[3];
    for (int c = 0; c < 3; ++c) {
        auto fl = std::make_shared<SPHParticles>(f, 400u);
        auto bd = std::make_shared<SPHParticles>(b);
        std::shared_ptr<BaseSolver> s;
        if (c == 0) s = std::make_shared<Other>();
        else if (c == 1) s = std::make_shared<DFSPHSolver>(static_cast<int>(f.size()));   // buffers smaller than the capacity
        else s = std::make_shared<DFSPHSolver>(400);
        SPHSystem sys(fl, bd, s, space, 0.0404f, 0.04f, 0.004f, 76.596750762082e-6f, 1.0f, 1.4f, 10.0f, 5e-4f, 1e-4f, 1e-4f, G, cells,
                      {}, ob);
        active[c] = sys.openBoundariesActive() ? 1 : 0;
    }
    std::printf("ACTIVE %d %d %d\n", active[0], active[1], active[2]);
    return 0;
}
"""


def test_class_layer_refusals(built, tmp_path):
    """a solver that is not a BasicSPHSolver, and one whose buffers are smaller than the capacity, get a closed system"""
    _gpu()
    src = tmp_path / "refusals.cpp"
    src.write_text(CLASS_REFUSALS)
    exe = str(tmp_path / "refusals")
    here = os.path.join(ROOT, "cpp-fluid-particles_b200")
    cmd = [shutil.which("g++") or "/usr/bin/g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(here, "host"),
           "-I/usr/local/cuda/include", "-o", exe, str(src), "-L" + here, "-lsphhost", "-lsphk", "-L/usr/local/cuda/lib64", "-lcudart",
           "-Wl,-rpath," + here, "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ACTIVE 0 0 1" in r.stdout, r.stdout
    assert r.stdout.count("open boundaries refused") == 2


# ---- 9. sph_headless --tap --drain with blocking launches (memcheck with SPHK_SANITIZER=1) ----------------------------------
@pytest.mark.parametrize("solver", ["sph", "dfsph", "pbd"])
def test_headless_runs_cleanly(built, tmp_path, solver):
    _gpu()
    cmd = [CLI, "--solver", solver, "--frames", "6", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055",
           "0.135", "--quiet", "--tap", "3.0", "--drain", "0.25", "--capacity", "2100"] + (["--iters", "2"] if solver != "sph" else []) + \
          (["--vorticity", "0.01"] if solver == "pbd" else [])
    env = dict(os.environ, SPHK_STEP_GRAPH="0")
    if os.environ.get("SPHK_SANITIZER") == "1":
        exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
        r = subprocess.run([exe, "--tool", "memcheck", "--error-exitcode", "9"] + cmd, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
        assert r.returncode == 0 and "ERROR SUMMARY: 0 errors" in r.stdout, r.stdout[-4000:]
        return
    prefix = str(tmp_path / "dump")
    env["CUDA_LAUNCH_BLOCKING"] = "1"
    r = subprocess.run(cmd + ["--dump", prefix], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-4000:]
    bad = [line for line in r.stdout.splitlines() if "failed" in line or "error" in line.lower()]
    assert not bad, "\n".join(bad[-20:])
    pos = np.fromfile(prefix + ".pos.f32", np.float32)
    assert pos.size > 0 and np.isfinite(pos).all()
    import json
    summary = json.loads(r.stdout.strip().splitlines()[-1])
    assert summary["open_check"] == 0 and summary["emitted"] > 0
