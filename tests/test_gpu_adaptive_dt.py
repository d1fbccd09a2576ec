"""CFL-adaptive time stepping on the GPU: the speed bound per element against numpy, fixed-dt systems unchanged by a bound that
never binds, every step's dt equal to the rule applied to the previous step's velocities, the DFSPH warm start across a dt
change, the layers (class layer through sph_headless and the facade, python engine) agreeing bit for bit, a fast block thrown at
a wall, and validation and refusals."""
import ctypes as C
import dataclasses
import json
import math
import os
import subprocess

import numpy as np
import pytest

import adaptive_dt_ref as AR
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
INVALID, STATE = -1, -4


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _np(t):
    return t.detach().cpu().numpy().copy()


def _same(a, b, what):
    for f in ("pos", "vel", "density", "pressure"):
        x, y = np.asarray(a[f]), np.asarray(b[f])
        assert x.shape == y.shape and np.array_equal(bits(x), bits(y)), f"{what}: {f} differs"


def _speed(s, vel, n, with_bodies=0):
    """sphk_step_speed over the first n rows of a (cap, 3) device tensor, then its result"""
    from cpp_fluid_particles_b200.engine import _ptr
    p = s.fluid.abi()
    p.vel, p.n = _ptr(vel), n
    assert s.L.sphk_step_speed(s.ctx, C.byref(p), C.c_int(with_bodies)) == 0
    v, bad = (C.c_float * 2)(), C.c_int(0)
    assert s.L.sphk_step_speed_result(s.ctx, v, C.byref(bad)) == 0
    return F(v[0]), F(v[1]), int(bad.value)


# ---- 1. the speed bound per element -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 33, 2 ** 21 + 1])
def test_speed_bound_per_element(pkg, built, n):
    """random, all-zero, NaN / +-inf in a few slots, and a set truncated below the array's length"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s = engine.SphkSystem(sc, step0=False, max_fluid=max(n, sc.fluid.shape[0]))
    rng = np.random.default_rng(n)
    base = rng.normal(0, 2.0, (n, 3)).astype(F)
    cases = {"random": base, "zero": np.zeros((n, 3), F)}
    bad = base.copy()
    for k, x in zip(rng.choice(n, min(n, 3), replace=False), (np.nan, np.inf, -np.inf)):
        bad[k, int(k) % 3] = x
    cases["nonfinite"] = bad
    big = base.copy()
    big[n - 1] = (50.0, 0.0, 0.0)          # the fastest particle sits in the last slot, outside a truncated set
    cases["truncated"] = big
    for name, v in cases.items():
        t = torch.from_numpy(v).to(s.device)
        m = n - 1 if name == "truncated" and n > 1 else n
        got, body, nonfin = _speed(s, t, m)
        want, wbad = AR.fluid_speed(v[:m])
        assert bits(np.array([got])) == bits(np.array([F(want)])) and nonfin == wbad and body == 0, (name, got, want, nonfin, wbad)
        if name == "nonfinite":
            assert wbad == min(n, 3)
    s.close()


def test_speed_bound_of_bodies(pkg, built):
    """|V| + |Omega| r_max per body from the device-resident motions, against float64; a non-finite motion cannot be set"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    rng = np.random.default_rng(3)
    bodies = []
    for b in range(5):
        pts = rng.uniform(-0.03, 0.03, (40 + b, 3)).astype(F)
        bodies.append({"points": pts, "position": (0.1 + 0.06 * b, 0.4, 0.35), "orientation": (0, 0, 0, 1),
                       "linear_velocity": rng.normal(0, 1, 3).astype(F), "angular_velocity": rng.normal(0, 20, 3).astype(F)})
    s = engine.SphkSystem(sc, step0=False, bodies=bodies)
    rmax = [float(np.sqrt((np.asarray(b["points"], np.float64) ** 2).sum(1)).max()) for b in bodies]
    zero = torch.zeros((s.fluid.pos.shape[0], 3), dtype=torch.float32, device=s.device)
    for trial in range(3):
        motion = s.current_body_motion()
        _, got, nonfin = _speed(s, zero, s.fluid.n, with_bodies=1)
        want = AR.body_speed64(motion, rmax)
        assert nonfin == 0 and abs(float(got) - want) <= 2e-6 * want, (got, want)
        # without the |Omega| r_max term the bound would be the largest |V| alone
        assert float(got) > float(np.linalg.norm(motion[:, :3], axis=1).max()) * 1.5
        s.set_body_motion(trial, rng.normal(0, 3, 3), rng.normal(0, 40, 3))
    _, got0, _ = _speed(s, zero, s.fluid.n, with_bodies=0)
    assert got0 == 0
    s.close()


# ---- 2. a bound that never binds changes nothing -------------------------------------------------------------------------------
def _throw_block(s, solver, speed):
    """the fluid block moving at `speed` along +x (PBD: through its last positions)"""
    n = s.fluid.n
    s.fluid.vel[:n, 0] = speed
    s.fluid.vel[:n, 1:] = 0
    if solver == "pbd":
        s.copy(s.pos_last, s.fluid.pos)
        s.pos_last[:n, 0] -= F(s.p.dt) * F(speed)


@pytest.mark.parametrize("solver", SOLVERS)
def test_never_binding_bound_changes_nothing(pkg, built, tmp_path, solver):
    """50 steps at C = 1e6 with dt_max = dt: the class layer's bits equal those of the fixed-dt system (with a dynamic body, and
    with an emitter); turning adaptivity off again brings the step graph back"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", solver)
    em = {"origin": (0.4, 0.42, 0.4), "direction": (0, -1, 0), "speed": 1.5, "spacing": 0.02, "width": 4, "height": 4}
    body = {"points": np.random.default_rng(0).uniform(-0.03, 0.03, (60, 3)).astype(F), "position": (0.4, 0.4, 0.4),
            "orientation": (0, 0, 0, 1), "linear_velocity": (0, 0, 0), "angular_velocity": (0, 0, 0), "mass": 0.05,
            "inertia": (1e-4, 1e-4, 1e-4)}
    n = sc.fluid.shape[0]
    for kw in ({}, {"bodies": [body]}, {"max_fluid": 2 * n, "emitters": [em], "sinks": []}):
        fixed, adapt = capi.SphApp(sc, **kw), capi.SphApp(sc, **kw)
        adapt.set_adaptive_dt(1e6, 0.0, float(sc.params.dt))
        for _ in range(50):
            fixed.step()
            adapt.step()
        _same(adapt.download(), fixed.download(), f"{solver} {list(kw)}")
        st = adapt.adaptive_stats()
        assert st["last_dt"] == F(sc.params.dt) and st["min_clamps"] == 0 and st["nonfinite_steps"] == 0
        assert not adapt.step_graph_active()
        if not kw:
            assert fixed.step_graph_active()
            adapt.set_adaptive_dt(0.0)
            for _ in range(3):
                adapt.step()
            assert adapt.step_graph_active()
        fixed.close()
        adapt.close()


# ---- 3. every dt is the rule's -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_each_dt_follows_the_rule(pkg, built, solver):
    """a block thrown at the wall (3 m/s; WCSPH, whose dt is 4 times smaller, 10 m/s): each step's dt is the reference rule
    applied to the velocities the previous step left"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", solver)
    s = engine.SphkSystem(sc)
    _throw_block(s, solver, 10.0 if solver == "wcsph" else 3.0)
    s.set_adaptive(0.2)
    r = s._rule
    prev = s.last_dt
    dts = []
    for _ in range(50):
        v, nonfin = AR.fluid_speed(_np(s.fluid.vel[:s.fluid.n]))
        s.step()
        want, _ = AR.rule(r.cfl, r.dt_min, r.dt_max, r.radius, r.gravity, float(v), prev, 0.0)
        assert s.last_dt == want and nonfin == 0
        prev = s.last_dt
        dts.append(prev)
    assert min(dts) < 0.8 * float(sc.params.dt)             # the bound binds at this speed
    assert s.simulated_time == math.fsum([float(F(sc.params.dt))] + dts)
    s.close()


# ---- 4. DFSPH's warm start across a dt change -----------------------------------------------------------------------------------
def test_dfsph_warm_start_is_independent_of_dt(pkg, built):
    """the warm-start correction moves a particle by dt * dv = sum m (k_i + k_j) gradW, whatever the dt of the step applying it"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene("mini", "dfsph", dt=0.004)
    s = engine.SphkSystem(sc)
    for _ in range(5):
        s.step()
    s.search_fluid()
    s.build_neighbor_list()
    s.permute(s.warm, 1)
    n = s.fluid.n
    s.warm[:n] = torch.from_numpy(np.random.default_rng(1).uniform(0, 1e-3, n).astype(F)).to(s.device)   # a warm start to apply
    v0 = torch.zeros_like(s.fluid.vel)        # from rest: the velocity after the sweep is the correction alone
    moved = []
    for dt in (0.004, 0.0013):
        s.fluid.vel.copy_(v0)
        s.refresh()
        s._step_dt = dt
        s.dfsph_den_correct(s.warm)
        moved.append(_np(s.fluid.vel[:s.fluid.n]).astype(np.float64) * float(F(dt)))
    s._step_dt = None
    scale = np.abs(moved[0]).max()
    assert scale > 0 and np.abs(moved[0] - moved[1]).max() <= 1e-5 * scale
    s.close()


# DFSPH across a dt change: the 9 execution paths of the engine (int32 lists with the staged and the global builder and with the
# per-particle overflow fallback, the cell walk, tile lists with and without overflow, and one kernel per launch site on lists,
# cells and tiles), each from the same state and warm start
DFSPH_PATHS = {"list": {}, "list_global": {"staged": 0}, "cap36": {"kmax": 36}, "cells": {"use_list": False}, "tile": {"tile": 1},
               "tile_cap36": {"tile": 1, "kmax": 36}, "unfused_list": {"fused": False}, "unfused_cells": {"fused": False, "use_list": False},
               "unfused_tile": {"fused": False, "tile": 1}}


def _dfsph_from(pkg, sc, st, warm, path, dt_b, warm_scale=1.0):
    """an engine system built from a state (already in search order) and its warm start, one step at dt_b along `path`"""
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    s = engine.SphkSystem(dataclasses.replace(sc, fluid=np.ascontiguousarray(st["pos"])), step0=False,
                          use_list=path.get("use_list", True), list_capacity=path.get("kmax", 96))
    s.set_option(capi.OPT_STAGED_LIST_BUILD, path.get("staged", 1))
    s.set_option(capi.OPT_TILE, path.get("tile", 0))
    s.fused = path.get("fused", True)
    n = s.fluid.n
    s.fluid.vel[:n] = torch.from_numpy(st["vel"]).to(s.device)
    s.warm[:n] = torch.from_numpy((warm * F(warm_scale)).astype(F)).to(s.device)
    s.set_adaptive(1e6, 0.0, dt_b)           # a bound that never binds: the step runs at dt_max = dt_b
    s.step()
    assert s.last_dt == F(dt_b)
    out = s.state()
    s.close()
    return out


def test_dfsph_step_across_a_dt_change_on_every_path(pkg, built):
    """a block thrown at the wall: 12 steps at dt_a = 4 ms build a warm start, then one step at dt_b = 1.3 ms from that state and
    warm start, on each of the 9 paths, equals the list path per element within the suite's tolerance; the same step with the warm
    start rescaled by dt_a / dt_b does not (the warm start is a displacement, DESIGN.md section 2.8)"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    from util import TOL, relerr
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s = engine.SphkSystem(sc)
    _throw_block(s, "dfsph", 4.0)
    for _ in range(12):
        s.step()
    s.search_fluid()                         # the state in search order, so the rebuilt systems' first search keeps it
    s.permute(s.warm, 1)
    st = s.state()
    warm = _np(s.warm[:s.fluid.n])
    s.close()
    assert np.abs(warm).max() > 0, "the block must be compressed against the wall: a warm start to carry across the change"
    dt_b = 0.0013
    ref = _dfsph_from(pkg, sc, st, warm, DFSPH_PATHS["list"], dt_b)
    for name, path in DFSPH_PATHS.items():
        got = _dfsph_from(pkg, sc, st, warm, path, dt_b)
        for f in ("pos", "vel", "density"):
            assert np.isfinite(got[f]).all() and relerr(got[f], ref[f]) <= TOL, (name, f, relerr(got[f], ref[f]))
    scaled = _dfsph_from(pkg, sc, st, warm, DFSPH_PATHS["list"], dt_b, warm_scale=0.004 / dt_b)
    assert relerr(scaled["vel"], ref["vel"]) > 100 * TOL


# PBD across a dt change: the velocity a step derives from positions, against numpy on read-back positions
def _pbd_probe_scene(pkg):
    """isolated particles (0.07 apart, more than the support radius R = 0.04, and away from the walls): the projection, XSPH and the
    surface terms leave them alone, so a step's velocity is the derived one plus dt G; and a 2 x 2 nozzle 0.05 apart"""
    sc = pkg.scene.benchmark_scene("mini", "pbd")
    g = np.arange(4, dtype=F) * F(0.07) + F(0.12)
    fluid = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(F)
    em = {"origin": (0.42, 0.42, 0.42), "direction": (0.0, -1.0, 0.0), "speed": 3.0, "spacing": 0.05, "width": 2, "height": 2}
    return dataclasses.replace(sc, fluid=fluid), em


@pytest.mark.parametrize("layer", ["class", "engine"])
def test_pbd_derives_velocity_over_the_previous_dt(pkg, built, layer):
    """the dt alternates between 4 and 1.3 ms.  Every particle's velocity after step k is (x_{k-1} - x_{k-2}) / dt_{k-1} + dt_k G
    from the read-back positions, and a layer emitted in step k moves at u d + dt_k G"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc, em = _pbd_probe_scene(pkg)
    G = np.asarray(sc.params.gravity, F)
    cap = sc.fluid.shape[0] + 400
    if layer == "class":
        sys_ = capi.SphApp(sc, max_fluid=cap, emitters=[em], sinks=[])
        read = lambda: sys_.download()  # noqa: E731

        def step(dt):
            sys_.set_adaptive_dt(1e6, 0.0, dt)
            sys_.step()
    else:
        sys_ = engine.SphkSystem(sc, max_fluid=cap, emitters=[em], sinks=[])
        read = lambda: sys_.state()  # noqa: E731

        def step(dt):
            sys_.set_adaptive(1e6, 0.0, dt)
            sys_.step()
    P, V, dts = [read()["pos"].copy()], [None], [None]     # after the constructor's step (it only initialises PBD's history)
    origin_of = [None]                                      # per step: index of each particle in the previous read-back (-1: emitted)
    emitted_checked = derived_checked = 0
    u_d = np.array([0.0, -3.0, 0.0], F)
    for k in range(1, 31):
        dt = 0.004 if k % 2 else 0.0013
        step(dt)
        st = read()
        pos, vel = st["pos"].copy(), st["vel"].copy()
        start = pos.astype(np.float64) - float(F(dt)) * vel.astype(np.float64)    # where each particle began the step
        d = np.linalg.norm(start[:, None, :] - P[-1][None, :, :].astype(np.float64), axis=2)
        j = d.argmin(1)
        org = np.where(d[np.arange(len(j)), j] < 1e-5, j, -1)
        a = F(dt) * G
        for i in range(len(pos)):
            if org[i] < 0:                                  # emitted in this step: its history was x - dt_{k-1} u d
                if k >= 2:
                    assert np.allclose(vel[i], u_d + a, rtol=0, atol=6e-4), (k, i, vel[i])
                    emitted_checked += 1
                continue
            l = origin_of[-1][org[i]] if origin_of[-1] is not None else -1
            if l < 0 or k < 2:
                continue
            want = (P[-1][org[i]] - P[-2][l]) / F(dts[-1]) + a
            assert np.allclose(vel[i], want, rtol=1e-5, atol=1e-6), (k, i, vel[i], want, dts[-1], dt)
            derived_checked += 1
        P.append(pos)
        V.append(vel)
        dts.append(dt)
        origin_of.append(org)
    assert derived_checked > 500 and emitted_checked >= 8, (derived_checked, emitted_checked)
    sys_.close()


def test_engine_adaptive_without_a_first_step(pkg, built):
    """step0=False, then adaptive: the first dt_prev is the scene's dt, as in the class layer"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s = engine.SphkSystem(sc, step0=False, adaptive={"C": 0.2})
    assert s.last_dt == F(sc.params.dt)
    s.step()
    assert s.advance(0.004) >= 1
    s.close()


def test_new_motion_sets_the_next_dt(pkg, built):
    """a body set spinning between steps, or fluid velocities uploaded between steps, bound the very next step's dt"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    body = {"points": np.random.default_rng(0).uniform(-0.03, 0.03, (60, 3)).astype(F), "position": (0.4, 0.4, 0.4),
            "orientation": (0, 0, 0, 1), "linear_velocity": (0, 0, 0), "angular_velocity": (0, 0, 0)}
    for layer in ("class", "engine"):
        sys_ = capi.SphApp(sc, bodies=[body]) if layer == "class" else engine.SphkSystem(sc, bodies=[body])
        if layer == "class":
            sys_.set_adaptive_dt(0.2)
        else:
            sys_.set_adaptive(0.2)
        sys_.step()
        sys_.set_body_motion(0, (6.0, 0.0, 0.0), (0.0, 0.0, 0.0))
        sys_.step()
        stats = sys_.adaptive_stats() if layer == "class" else sys_.adaptive_stats
        last = stats["last_dt"] if layer == "class" else sys_.last_dt
        assert stats["source"] == 1 and abs(stats["speed"] - 6.0) < 1e-6, (layer, stats)
        assert last < 0.2 * 0.04 / 6.0 * 1.0001, (layer, last)
        sys_.close()
    app = capi.SphApp(sc)
    app.set_adaptive_dt(0.2)
    app.step()
    st = app.download()
    vel = st["vel"].copy()
    vel[0] = (8.0, 0.0, 0.0)
    app.upload(vel=vel)
    app.step()
    a = app.adaptive_stats()
    assert a["source"] == 0 and a["speed"] >= 8.0 and a["last_dt"] < 0.2 * 0.04 / 8.0 * 1.0001, a
    app.close()


# ---- 5. the layers agree -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver,extra", [("wcsph", []), ("dfsph", []), ("pbd", []), ("dfsph", ["--tap", "2.5"]),
                                          ("pbd", ["--tap", "2.5"]), ("dfsph", ["--float", "0.6"]), ("wcsph", ["--float", "0.6"])])
def test_layers_agree(pkg, built, tmp_path, solver, extra):
    """sph_headless --cfl, the facade and the python engine: the same substeps and bits after 20 frames; simulated time is the
    double sum of the float dts"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    prefix = str(tmp_path / "s")
    base = [CLI, "--solver", solver, "--iters", "4", "--box", str(box), "--block", str(nx), str(ny), str(nz), "--origin",
            *[repr(float(o)) for o in origin]] + extra
    r = subprocess.run(base + ["--emit-scene", prefix], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    fluid = np.fromfile(prefix + ".fluid.f32", F).reshape(-1, 3)
    sc = dataclasses.replace(pkg.scene.benchmark_scene("mini", solver), fluid=fluid)
    kw = {}
    if "--tap" in extra:
        ev = np.fromfile(prefix + ".emitter.f32", F)
        kw = {"max_fluid": 2 * fluid.shape[0], "sinks": [],
              "emitters": [{"origin": ev[:3], "direction": ev[3:6], "speed": ev[6], "spacing": ev[7], "width": int(ev[8]),
                            "height": int(ev[9])}]}
    if "--float" in extra:
        bs, dyn = np.fromfile(prefix + ".body_state.f32", F), np.fromfile(prefix + ".body_dyn.f32", F)
        kw = {"bodies": [{"points": np.fromfile(prefix + ".body.f32", F).reshape(-1, 3), "position": bs[:3], "orientation": bs[3:7],
                          "linear_velocity": bs[7:10], "angular_velocity": bs[10:13], "mass": dyn[0], "inertia": dyn[1:4]}]}
    C_ = 0.05                # small enough that dt changes from step to step in every variant
    s = engine.SphkSystem(sc, adaptive={"C": C_}, **kw)
    app = capi.SphApp(sc, **kw)
    app.set_adaptive_dt(C_)
    frames, dt = 20, float(sc.params.dt)
    ks = []
    for _ in range(frames):
        k = s.advance(dt)
        assert app.advance(dt) == (k, F(s.adaptive_stats["frame_min_dt"]))
        ks.append(k)
    st = s.state()
    _same(app.download(), st, f"{solver} {extra}: facade vs engine")
    a = app.adaptive_stats()
    assert a["simulated_time"] == s.simulated_time and a["last_dt"] == s.last_dt
    assert abs(s.simulated_time - (frames + 1) * dt) <= (frames + 1) * float(np.spacing(F(dt)))
    app.close()
    r = subprocess.run(base + ["--cfl", str(C_), "--frames", str(frames), "--quiet", "--dump", prefix], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    pos = np.fromfile(prefix + ".pos.f32", F).reshape(-1, 3)
    assert np.array_equal(bits(pos), bits(st["pos"])), "sph_headless"
    assert np.isfinite(pos).all()
    summary = json.loads(r.stdout.strip().splitlines()[-1])
    assert summary["frame_substeps"] == ks and summary["simulated_time"] == s.simulated_time
    assert sum(ks) >= frames
    s.close()


# ---- 6. physics: a block thrown at the wall ------------------------------------------------------------------------------------
SPEED = 4.0            # m/s along +x, towards the wall 0.18 away
WALL_GAP = 0.01        # every fluid particle stays this far (half a spacing) inside the wall layer at x = 0.995 L
COMPRESSION_BOUND = 0.3   # max (rho / rho0 - 1) the adaptive run stays under (DESIGN.md section 2.8)


@pytest.mark.parametrize("solver", ["dfsph", "pbd"])
def test_block_thrown_at_the_wall(pkg, built, solver):
    """the adaptive run keeps every particle in the clamp box and off the wall layer, and its compression under the bound"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", solver)
    s = engine.SphkSystem(sc)
    _throw_block(s, solver, SPEED)
    s.set_adaptive(0.2)
    worst = 0.0
    space = np.asarray(sc.params.space, np.float64)
    wall = 0.995 * space[0]
    for _ in range(40):
        s.advance(float(sc.params.dt))
        st = s.state()
        pos, den = st["pos"].astype(np.float64), st["density"].astype(np.float64)
        assert np.isfinite(pos).all() and (pos >= 0).all() and (pos <= 0.99 * space + 1e-6).all()
        assert pos[:, 0].max() <= wall - WALL_GAP, pos[:, 0].max()
        worst = max(worst, float((den / sc.params.rho0 - 1).max()))
    assert worst < COMPRESSION_BOUND, worst
    s.close()


# ---- 7. validation and refusals -------------------------------------------------------------------------------------------------
def test_validation_and_refusals(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s = engine.SphkSystem(sc, step0=False)
    L, ctx = s.L, s.ctx
    p = s.fluid.abi()
    v, bad = (C.c_float * 2)(), C.c_int(0)
    assert L.sphk_step_speed_result(ctx, v, C.byref(bad)) == STATE            # before the first bound
    assert L.sphk_step_speed(ctx, C.byref(p), 1) == STATE                      # no bodies
    q = s.fluid.abi()
    q.n = -1
    assert L.sphk_step_speed(ctx, C.byref(q), 0) == INVALID
    q.n = s.fluid.pos.shape[0] + 1
    assert L.sphk_step_speed(ctx, C.byref(q), 0) == INVALID
    q = s.fluid.abi()
    q.vel = None
    assert L.sphk_step_speed(ctx, C.byref(q), 0) == INVALID
    assert L.sphk_set_active_range(ctx, 0, 10) == 0
    assert L.sphk_step_speed(ctx, C.byref(p), 0) == STATE                      # slab ranks
    assert L.sphk_set_active_range(ctx, 0, -1) == 0
    assert L.sphk_step_speed(ctx, C.byref(p), 0) == 0
    assert L.sphk_step_speed_result(ctx, v, None) == INVALID
    for args in ((0.0,), (-0.2,), (float("nan"),), (0.2, -1.0), (0.2, float("inf")), (0.2, 0.01, 0.001)):
        with pytest.raises(ValueError):
            s.set_adaptive(*args)
    assert not s.adaptive
    with pytest.raises(ValueError):
        s.advance(0.004)                                                        # not adaptive
    s.set_adaptive(0.2)
    with pytest.raises(ValueError):
        s.advance(float("nan"))
    s.close()
    app = capi.SphApp(sc)
    for args in ((-0.2,), (float("nan"),), (0.2, -1.0, 0.0), (0.2, 0.01, 0.001), (float("inf"),)):
        with pytest.raises(RuntimeError):
            app.set_adaptive_dt(*args)
    with pytest.raises(RuntimeError):
        app.advance(0.004)                                                      # not adaptive
    app.set_adaptive_dt(0.2)
    with pytest.raises(RuntimeError):
        app.set_adaptive_dt(0.2, 0.01, 0.001)                                   # refused, the setting kept
    for T in (0.0, -1.0, float("inf")):
        with pytest.raises(RuntimeError):
            app.advance(T)
    pos = np.zeros((app.nF, 3), F)
    with pytest.raises(RuntimeError):
        app.submit(pos, pos)                                                    # the pipelining assumes a fixed step
    assert app.advance(0.004)[0] >= 1
    app.close()
    em = {"origin": (0.4, 0.42, 0.4), "direction": (0, -1, 0), "speed": 1.5, "spacing": 0.02, "width": 4, "height": 4}
    n = sc.fluid.shape[0]
    app = capi.SphApp(sc, max_fluid=2 * n, emitters=[em], sinks=[])
    with pytest.raises(RuntimeError):
        app.set_adaptive_dt(0.2, 0.0, 2 * float(sc.params.dt))     # the emitters were checked for the constructor's dt
    app.set_adaptive_dt(0.2, 0.0, float(sc.params.dt))
    app.close()
    s = engine.SphkSystem(sc, max_fluid=2 * n, emitters=[em], sinks=[])
    with pytest.raises(ValueError):
        s.set_adaptive(0.2, 0.0, 2 * float(sc.params.dt))
    assert not s.adaptive
    s.close()
