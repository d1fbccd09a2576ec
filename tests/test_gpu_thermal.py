"""Heat transfer on the GPU: the conduction sweep per element on every execution path against the float64 reference
(tests/thermal_ref.py), walls and a body at their own temperatures, the statistics and the fixed-shape reduction, conservation,
the maximum principle, the decay rate of a cosine profile, buoyancy, the temperature-dependent viscosity, non-interference, the
step graph and the layers."""
import numpy as np
import pytest

import ref64
import sweep_driver as SD
import test_gpu_implicit_viscosity as TIV
import thermal_ref as TR
from util import bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
_gpu, _np, _case, _system, _app, _same = TIV._gpu, TIV._np, TIV._case, TIV._system, TIV._app, TIV._same


def _temperature(pos):
    return (20.0 + 30.0 * np.sin(9.0 * pos[:, 0]) * np.cos(7.0 * pos[:, 1]) + 10.0 * pos[:, 2]).astype(F)


# ---- 1. the conduction sweep per element on every path ----------------------------------------------------------------------
@pytest.mark.parametrize("path", sorted(SD.PATHS))
@pytest.mark.parametrize("scene", ["config0", "config0_mass", "walls", "n33", "body", "body_without_entry"])
def test_conduction_per_element(pkg, built, scene, path):
    """dT/dt against float64; the statistics at a substep dt that puts about half the particles above the stability bound (the
    count is exact away from the rounding band around 1).  body_without_entry: hot walls and no entry for the body, whose
    particles must then be adiabatic"""
    _gpu()
    import torch
    case, bodies = _case(pkg, scene.split("_")[0])
    s, P, _, _ = _system(pkg, case, bodies, SD.PATHS[path])
    p = case.sc.params
    n = s.fluid.n
    try:
        T = _temperature(s.state()["pos"])
        groups = [(80.0, 1.0)] + ([(-15.0, 2.5)] if scene == "body" else [])
        spec = dict(alpha=1e-3, beta=0.0, t_ref=20.0, wall=groups[0], bodies=groups[1:])
        gB = _np(s.body_local())[:, 3].astype(np.int64) if bodies else None
        ref = TR.conduction(P, T, spec["alpha"], p.rho0, p.rho_boundary, gB, groups)
        if scene == "body_without_entry":
            wall_only = TR.conduction(P, T, spec["alpha"], p.rho0, p.rho_boundary, None, groups)
            assert np.abs(wall_only["value"] - ref["value"]).max() > 1e-3 * np.abs(ref["value"]).max(), "the body touches no fluid"
        dt_sub = float(F(1.0 / np.median(ref["csum"][ref["csum"] > 0]))) if n > 1 else 1e-3
        tg = torch.from_numpy(T).to(s.device)
        out = torch.zeros(n, dtype=torch.float32, device=s.device)
        s.heat_conduction(tg, out, dt_sub, spec)
        got = _np(out)
        ref64.assert_per_element(got, ref64.R64(ref["value"], ref["mag"]), ref64.TAU, f"{scene}/{path} dT/dt", ref64.f32_spacing(got))
        st = s.thermal_stats()
        cour = dt_sub * ref["csum"]
        cmax = cour.max()
        assert abs(st["max_courant"] - cmax) <= 1e-5 * cmax + 1e-30, (st["max_courant"], cmax)
        lo, hi = int((cour > 1.0 + 1e-5).sum()), int((cour > 1.0 - 1e-5).sum())
        assert lo <= st["violators"] <= hi, (st["violators"], lo, hi)
        if n > 100:
            assert lo > 0.2 * n, "the statistics case has no violators"
        if scene == "body":     # the body's group and its own temperature reach the fluid
            assert (P.jB.size > 0) and np.any(gB[P.jB] > 0)
    finally:
        s.close()


def test_buoyancy_per_element(pkg, built):
    """the last substep's dv = -beta (T - T_ref) G dt on the API velocities and the records, against float64 (alpha = 0: T stays)"""
    _gpu()
    import ctypes as C
    import torch
    from cpp_fluid_particles_b200 import capi
    case, bodies = _case(pkg, "config0")
    s, _, _, _ = _system(pkg, case, bodies)
    p = case.sc.params
    n = s.fluid.n
    try:
        rng = np.random.default_rng(5)
        v0 = (0.3 * rng.standard_normal((n, 3))).astype(F)
        TIV._set_vel(s, v0)
        T = _temperature(s.state()["pos"])
        T[::7] = F(20.0)                                  # some particles at T_ref: no write at all
        th = capi.thermal(dict(alpha=0.0, beta=0.013, t_ref=20.0))
        t, work = torch.from_numpy(T).cuda(), torch.zeros(n, dtype=torch.float32, device=s.device)
        g = (C.c_float * 3)(0.3, -9.8, 0.1)
        dt = float(F(0.004))
        for k in range(3):
            assert s.L.sphk_heat_step(s.ctx, s._s(), C.byref(th), C.c_void_p(t.data_ptr()), C.c_void_p(work.data_ptr()), C.c_float(dt),
                                      C.c_int(k), C.c_int(3), C.c_float(p.rho0), C.c_float(p.rho_boundary), g) == 0
        v = _np(s.fluid.vel)
        dT = T.astype(np.float64) - np.float64(F(20.0))
        ref = v0 - (float(F(0.013)) * dT)[:, None] * (np.array([F(0.3), F(-9.8), F(0.1)], np.float64) * dt)[None]
        err = np.abs(v - ref) / (np.abs(v0) + np.abs(ref - v0) + 1e-30)
        assert err.max() < 4e-7, err.max()
        assert np.array_equal(bits(v[::7]), bits(v0[::7]))
        assert np.array_equal(_np(t), T)
    finally:
        s.close()


def test_heat_stats_reduction(pkg, built):
    """min T, max T and sum m T of sphk_heat_stats against numpy on sizes past one block and past the 1024-block cap"""
    _gpu()
    import torch
    s, _, _, _ = _system(pkg, *_case(pkg, "config0"))
    try:
        for n in (1, 255, 2049, 1024 * 2048 + 5):
            rng = np.random.default_rng(n)
            T = rng.uniform(-50, 200, n).astype(F)
            m = rng.uniform(0.5, 2.0, n).astype(F)
            t, mm = torch.from_numpy(T).cuda(), torch.from_numpy(m).cuda()
            import ctypes as C
            lo, hi, q = C.c_float(0), C.c_float(0), C.c_double(0)
            assert s.L.sphk_heat_stats(s.ctx, C.c_void_p(t.data_ptr()), C.c_void_p(mm.data_ptr()), C.c_int(n), None, None, C.byref(lo),
                                       C.byref(hi), C.byref(q)) == 0
            assert lo.value == T.min() and hi.value == T.max()
            ref = np.sum(m.astype(np.float64) * T.astype(np.float64))
            assert abs(q.value - ref) <= 1e-12 * np.sum(np.abs(m.astype(np.float64) * T)), (q.value, ref)
    finally:
        s.close()


# ---- 2. conservation, maximum principle, decay -----------------------------------------------------------------------------
def _rest_system(pkg, solver="dfsph", scene="mini"):
    """the mini block without gravity: a fluid at rest"""
    import dataclasses
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene(scene, solver)
    sc = dataclasses.replace(sc, params=dataclasses.replace(sc.params, gravity=(0.0, 0.0, 0.0)))
    return engine.SphkSystem(sc)


def test_adiabatic_walls_conserve_heat(pkg, built):
    _gpu()
    import torch
    s = _rest_system(pkg)
    try:
        s.thermal = dict(alpha=2e-3, beta=0.0, t_ref=0.0)
        n = s.fluid.n
        s.temperature[:n] = torch.from_numpy(_temperature(s.state()["pos"])).cuda()
        q0 = s.thermal_stats()["heat"]
        spread0 = float(s.temperature[:n].std())
        for _ in range(200):
            s.step()
        st = s.thermal_stats()
        m = s.state()["mass"].astype(np.float64)
        scale = float(np.sum(m * np.abs(_np(s.temperature[:n]))))
        assert abs(st["heat"] - q0) <= 200 * 4 * 6e-8 * scale, (st["heat"], q0)
        assert float(s.temperature[:n].std()) < 0.9 * spread0, "no conduction happened"
        assert st["violators"] == 0
    finally:
        s.close()


def test_maximum_principle_with_hot_walls(pkg, built):
    _gpu()
    import torch
    s = _rest_system(pkg)
    try:
        s.thermal = dict(alpha=2e-3, beta=0.0, t_ref=0.0, wall=(100.0, 1.0))
        n = s.fluid.n
        T0 = _temperature(s.state()["pos"])
        s.temperature[:n] = torch.from_numpy(T0).cuda()
        lo, hi = min(T0.min(), 100.0), max(T0.max(), 100.0)
        for _ in range(50):
            s.step()
            st = s.thermal_stats()
            assert st["violators"] == 0 and st["max_courant"] <= 1.0
            assert lo <= st["t_min"] and st["t_max"] <= hi, (st, lo, hi)
    finally:
        s.close()


def test_cosine_profile_decays_at_the_float64_rate(pkg, built):
    """T = cos(pi x / L) across the block at rest (adiabatic walls): its amplitude decays as in the float64 run of the same scene,
    and near alpha pi^2 / L^2"""
    _gpu()
    import torch
    from oracle import oracle as O
    s = _rest_system(pkg)
    try:
        alpha, steps = 2e-3, 40
        s.thermal = dict(alpha=alpha, beta=0.0, t_ref=0.0)
        st = s.state()
        x = st["pos"][:, 0]
        L = x.max() - x.min()
        T0 = np.cos(np.pi * (x - x.min()) / L).astype(F)
        n = s.fluid.n
        s.temperature[:n] = torch.from_numpy(T0).cuda()
        p = s.p
        g = O.grid(p.cell_size, p.cell_length, hash_rcp=s.device_rcp(p.cell_length))
        A = O.SceneArrays(st["pos"], st["mass"], st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius)
        P = ref64.Pairs(A)
        T64 = TR.run(P, T0, alpha, p.rho0, p.rho_boundary, p.dt, steps)
        for _ in range(steps):
            s.step()
        pos = s.state()["pos"]          # (the block relaxes by a fraction of a spacing; the float64 run keeps the first positions)
        Tg = _np(s.temperature[:n])
        amp = lambda t, xx: np.dot(t, np.cos(np.pi * (xx - x.min()) / L)) / np.dot(T0, T0)  # noqa: E731
        a_gpu, a64 = amp(Tg, pos[:, 0]), amp(T64, x)
        rate64 = -np.log(a64) / (steps * p.dt)
        print(f"\ncosine decay rate: float64 {rate64:.4f}, gpu {-np.log(a_gpu) / (steps * p.dt):.4f}, alpha pi^2/L^2 "
              f"{alpha * np.pi ** 2 / L ** 2:.4f}")
        assert abs(a_gpu - a64) <= 0.1 * (1 - a64), (a_gpu, a64)
        assert 0.5 < rate64 / (alpha * np.pi ** 2 / L ** 2) < 1.5
    finally:
        s.close()


# ---- 3. non-interference, graph, layers -------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_uniform_reference_temperature_changes_nothing(pkg, built, solver):
    """T = T_ref everywhere with adiabatic walls, any alpha and beta: the bits of thermal off; off and set-then-cleared launch
    what the parent launches"""
    _gpu()
    a, b, c = _app(pkg, solver), _app(pkg, solver), _app(pkg, solver)
    b.set_thermal(dict(alpha=5e-3, beta=0.7, t_ref=25.0))
    c.set_thermal(dict(alpha=5e-3, beta=0.7, t_ref=25.0)); c.set_thermal(None)
    try:
        for k in range(6):
            for x in (a, b, c):
                x.step()
            ra = a.download()
            _same(ra, b.download(), f"{solver} step {k} uniform T_ref")
            _same(ra, c.download(), f"{solver} step {k} set then cleared")
            assert np.all(b.download_temperature() == F(25.0))
    finally:
        for x in (a, b, c):
            x.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_graph_and_layers_agree(pkg, built, solver):
    """graph on and off give the same bits with heat transfer on; the facade and the python engine agree bit for bit"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    spec = dict(alpha=3e-3, beta=0.02, t_ref=20.0, wall=(60.0, 0.5))
    g, p = _app(pkg, solver), _app(pkg, solver)
    p.set_option(3, 0)
    e = engine.SphkSystem(pkg.scene.benchmark_scene("mini", solver))
    try:
        T0 = _temperature(g.download()["pos"])
        for x in (g, p):
            x.set_thermal(spec)
            x.upload_temperature(T0)
        e.thermal = spec
        e.temperature[:e.fluid.n] = torch.from_numpy(T0).cuda()
        for k in range(8):
            g.step(); p.step(); e.step()
            rg = g.download()
            _same(rg, p.download(), f"{solver} step {k}: graph vs plain")
            assert np.array_equal(bits(g.download_temperature()), bits(p.download_temperature()))
            _same(rg, e.state(), f"{solver} step {k}: facade vs engine", ("pos", "density"))
            assert np.array_equal(bits(g.download_temperature()), bits(_np(e.temperature[:e.fluid.n]))), f"{solver} step {k} T"
        assert g.step_graph_active() and not p.step_graph_active()
        assert g.thermal_stats()["substeps"] >= 1
    finally:
        g.close(); p.close(); e.close()


# ---- 4. physics ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["dfsph", "pbd"])
def test_hot_blob_rises(pkg, built, solver):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    cold, hot = [engine.SphkSystem(pkg.scene.benchmark_scene("mini", solver)) for _ in range(2)]
    try:
        for _ in range(10):
            cold.step(); hot.step()
        pos = hot.state()["pos"]
        c = pos.mean(0)
        blob = np.linalg.norm(pos - c, axis=1) < 0.05
        cold.thermal = dict(alpha=1e-4, beta=0.0, t_ref=20.0)      # the same tracer without buoyancy
        hot.thermal = dict(alpha=1e-4, beta=0.02, t_ref=20.0)
        T = np.where(blob, 80.0, 20.0).astype(F)
        for s in (cold, hot):
            s.temperature[:s.fluid.n] = torch.from_numpy(T).cuda()
        for _ in range(30):
            cold.step(); hot.step()
        # follow the blob by temperature (the particles are re-sorted every step)
        y = {}
        for name, s in (("cold", cold), ("hot", hot)):
            t, ps = _np(s.temperature[:s.fluid.n]), s.state()["pos"]
            warm = t > 50.0
            assert warm.sum() > 0.5 * blob.sum()
            y[name] = ps[warm, 1].mean()
        rise = y["hot"] - y["cold"]
        print(f"\n{solver}: hot blob centroid above the unheated tracer by {rise:.4f}")
        assert rise > 0.002
    finally:
        cold.close(); hot.close()


def test_thermal_viscosity_eval_and_e0_is_the_constant_solve(pkg, built):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "dfsph"))
    try:
        T = np.concatenate([np.linspace(-100, 300, 4001), [np.nan, 1e30, -1e30]]).astype(F)
        spec = dict(nu_ref=0.05, e=0.03, nu_min=1e-3, nu_max=2.0)
        nu = torch.zeros(T.size, dtype=torch.float32, device=s.device)
        s.thermal_viscosity_eval(spec, 20.0, torch.from_numpy(T).cuda(), nu)
        ref = TR.nu_of_t(T, *[float(F(x)) for x in (0.05, 0.03, 20.0, 1e-3, 2.0)]).astype(F)   # the law's float32 parameters
        assert np.array_equal(_np(nu), ref)
    finally:
        s.close()
    # E = 0: nu(T) = nu_ref everywhere, wall factor 1 -> the constant-nu solve with nu = nu_b = nu_ref, bit for bit
    a, b = _app(pkg, "dfsph"), _app(pkg, "dfsph")
    try:
        a.set_implicit_viscosity(0.05, 0.05)
        b.set_thermal(dict(alpha=0.0, beta=0.0, t_ref=20.0))
        b.set_thermal_viscosity(dict(nu_ref=0.05, e=0.0, nu_max=1.0, wall_factor=1.0))
        for k in range(4):
            a.step(); b.step()
            _same(a.download(), b.download(), f"step {k}: nu(T) with E = 0 vs the constant-nu solve")
    finally:
        a.close(); b.close()


def test_hot_block_runs_out_further(pkg, built):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    spread = {}
    for name, T in (("cold", 0.0), ("hot", 100.0)):
        s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "dfsph"))
        try:
            s.thermal = dict(alpha=0.0, beta=0.0, t_ref=0.0)
            s.thermal_viscosity = dict(nu_ref=0.5, e=0.05, nu_min=1e-3, nu_max=0.5, wall_factor=1.0)
            s.temperature.fill_(T)
            for _ in range(30):
                s.step()
            pos = s.state()["pos"]
            spread[name] = float(np.abs(pos[:, [0, 2]] - pos[:, [0, 2]].mean(0)).mean())
        finally:
            s.close()
    print(f"\nspread cold {spread['cold']:.4f} hot {spread['hot']:.4f}")
    assert spread["hot"] > spread["cold"]


def test_refusals(pkg, built):
    _gpu()
    import ctypes as C
    from cpp_fluid_particles_b200 import capi
    app = _app(pkg, "dfsph")
    try:
        with pytest.raises(RuntimeError):
            app.set_thermal(dict(alpha=-1.0))
        with pytest.raises(RuntimeError):
            app.set_thermal(dict(alpha=1.0, wall=(0.0, -1.0)))
        app.set_rheology(dict(model="cross", nu0=0.1, nu_inf=0.01, lam=1.0, m=1.0, nu_max=0.1))
        with pytest.raises(RuntimeError):
            app.set_thermal_viscosity(dict(nu_ref=0.1, e=0.0, nu_max=1.0))
    finally:
        app.close()
    L = capi.sphk()
    t = capi.thermal(dict(alpha=1.0, bodies=[(1.0, 1.0)]))
    k = C.c_int(0)
    assert L.sphk_heat_substeps(C.byref(t), C.c_float(0.04), C.c_float(1e-3), C.byref(k)) == 0
    assert k.value == TR.substeps(1.0, 1.0, 0.04, float(F(1e-3)))
    t.alpha = float("nan")
    assert L.sphk_heat_substeps(C.byref(t), C.c_float(0.04), C.c_float(1e-3), C.byref(k)) != 0


# ---- 5. carrying, open boundaries, adaptive dt --------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_every_particle_keeps_its_temperature(pkg, built, solver):
    """alpha = beta = 0 and T = f(x0): through 20 sorted steps of the dam break each particle keeps its own T, so |T - f(x)| stays
    within Lip(f) times the distance any particle can have moved"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", solver))
    try:
        s.step()
        s.thermal = dict(alpha=0.0, beta=0.0, t_ref=0.0)
        a = np.array([3.0, 2.0, -1.0])
        n = s.fluid.n
        st = s.state()
        s.temperature[:n] = torch.from_numpy((st["pos"].astype(np.float64) @ a).astype(F)).cuda()
        travel = 0.0
        for _ in range(20):
            v = s.state()["vel"]
            s.step()
            travel += float(np.linalg.norm(s.state()["vel"], axis=1).max() + np.linalg.norm(v, axis=1).max()) * 0.5 * s.dt
        pos = s.state()["pos"].astype(np.float64)
        err = np.abs(_np(s.temperature[:n]) - pos @ a)
        print(f"\n{solver}: max |T - f(x)| {err.max():.4f}, bound {np.linalg.norm(a) * 1.5 * travel:.4f}")
        assert err.max() <= np.linalg.norm(a) * 1.5 * travel + 1e-4
        assert travel > 0.002
    finally:
        s.close()


@pytest.mark.parametrize("layer", ["class", "engine"])
@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
def test_emitted_particles_carry_their_emitter_temperature(pkg, built, solver, layer):
    """alpha = 0: every emitted particle is at the emitter's 90, every original one at T_ref = 20; a sink in a corner of the block
    removes originals only, so the counts are the emitted count and the original count minus the removed"""
    _gpu()
    import test_gpu_open_boundaries as TOB
    from cpp_fluid_particles_b200 import capi, engine
    sc, em, sinks = TOB._open_scene(pkg, solver)
    n0 = sc.fluid.shape[0]
    cap = n0 + 600
    spec = dict(alpha=0.0, beta=0.0, t_ref=20.0, emitters=[90.0])
    if layer == "class":
        s = capi.SphApp(sc, max_fluid=cap, emitters=[em], sinks=sinks[:1])
        s.set_thermal(spec)
        temps = s.download_temperature
        stats = lambda: s.open_boundary_stats()[0]  # noqa: E731
    else:
        s = engine.SphkSystem(sc, max_fluid=cap, emitters=[em], sinks=sinks[:1])
        s.thermal = spec
        temps = lambda: _np(s.temperature[:s.fluid.n])  # noqa: E731
        stats = s.open_boundary_stats
    try:
        e0, r0 = stats()["emitted"], stats()["removed"]
        n_start = s.fluid_count
        for _ in range(12):
            s.step()
        st = stats()
        t = temps()
        emitted, removed = st["emitted"] - e0, st["removed"] - r0
        assert emitted > 0 and (removed > 0 or solver == "wcsph")   # (WCSPH's block does not reach the sink within the run)
        assert int((t == F(90.0)).sum()) == emitted
        assert int((t == F(20.0)).sum()) == n_start - removed
        assert t.size == n_start + emitted - removed
    finally:
        s.close()


def test_adaptive_dt_changes_the_substep_count(pkg, built):
    """an adaptive DFSPH system with a diffusivity whose substep count depends on dt: the count changes from step to step, every
    substep keeps the maximum principle and sum m T is conserved (adiabatic walls)"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.make_scene("mini", "dfsph", dt=0.004))
    try:
        s.set_adaptive(0.05)
        s.thermal = dict(alpha=0.02, beta=0.0, t_ref=0.0)
        n = s.fluid.n
        T0 = _temperature(s.state()["pos"])
        s.temperature[:n] = torch.from_numpy(T0).cuda()
        q0 = s.thermal_stats()["heat"]
        counts = []
        for _ in range(30):
            s.step()
            st = s.thermal_stats()
            counts.append(st["substeps"])
            assert st["violators"] == 0 and st["max_courant"] <= 1.0
            assert T0.min() <= st["t_min"] and st["t_max"] <= T0.max()
        m = s.state()["mass"].astype(np.float64)
        assert abs(st["heat"] - q0) <= 1e-5 * float(np.sum(m * np.abs(T0)))
        print(f"\nsubsteps of the last steps: {counts}")
        assert len(set(counts)) > 1, counts
    finally:
        s.close()


# ---- 6. the headless app -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["sph", "dfsph", "pbd"])
@pytest.mark.parametrize("extra,lo_hi", [(["--heat", "0.002,0.02,20", "--heater", "80"], (20.0, 80.0)),
                                         (["--heat", "0.002,0,0", "--heater", "100", "--thermal-viscosity", "0.5,0.05,5"], (0.0, 100.0)),
                                         (["--heat", "0.002,0.02,20", "--wall-temp", "5,1", "--tap", "2", "--tap-temp", "60", "--drain",
                                           "0.3"], (5.0, 60.0))])
def test_headless_heat_runs(built, tmp_path, solver, extra, lo_hi):
    """the heater, the melting block and a hot tap with cold walls run with blocking launches, print a heat line per frame and end
    with finite particles and temperatures inside the range of their sources"""
    import os
    import re
    import subprocess
    _gpu()
    cmd = [TIV.CLI, "--solver", solver, "--frames", "3", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.1",
           "0.135"] + (["--iters", "2"] if solver != "sph" else []) + extra
    env = dict(os.environ, SPHK_STEP_GRAPH="0", CUDA_LAUNCH_BLOCKING="1")
    prefix = str(tmp_path / "dump")
    r = subprocess.run(cmd + ["--dump", prefix], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-4000:]
    bad = [line for line in r.stdout.splitlines() if "failed" in line or "error" in line.lower()]
    assert not bad, "\n".join(bad[-20:])
    heat = [line for line in r.stdout.splitlines() if " heat - T min" in line]
    assert len(heat) == 3, r.stdout[-3000:]
    lo, hi = (float(x) for x in re.search(r"T min (\S+) max (\S+)", heat[-1]).groups())
    assert lo_hi[0] - 1e-3 <= lo <= hi <= lo_hi[1] + 1e-3, heat[-1]
    assert re.search(r", 0 above the stability bound", heat[-1]), heat[-1]
    pos = np.fromfile(prefix + ".pos.f32", np.float32)
    assert pos.size > 0 and np.isfinite(pos).all()
