"""Fluid-solid adhesion on the GPU: the sweep per element on every execution path against the float64 reference
(tests/adhesion_ref.py), bit-identical across the paths, the statistics, momentum with a dynamic body (also after the fluid moved
since the search), non-interference, the step graph and the layers, the footprint of a settling block, combinations with other
features, and the headless app."""
import json
import os
import subprocess

import numpy as np
import pytest

import adhesion_ref as AR
import ref64
import sweep_driver as SD
import test_gpu_implicit_viscosity as TIV
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
_gpu, _np, _system, _app, _same = TIV._gpu, TIV._np, TIV._system, TIV._app, TIV._same
WALL, BODY = 150.0, 90.0


def _case(pkg, scene):
    if scene.startswith("body"):
        return TIV._case(pkg, "body")
    return SD.make_case(pkg, scene), None


def _off_grid(s, pos):
    p = s.p
    c = np.trunc(pos.astype(np.float64) / np.float64(F(p.cell_length)))
    return np.any((c < 0) | (c >= np.asarray(p.cell_size)[None, :]), 1)


# ---- 1. the sweep per element on every path ----------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["config0", "config0_mass", "walls", "body", "body_without_entry"])
def test_accel_per_element_on_every_path(pkg, built, scene):
    """a_i against float64 (walls at 150, the body at 90 or without an entry); the same bits on all paths; the wetted count within
    the rounding bands at R/2 and R; the largest |a_i| is that of the per-element output"""
    _gpu()
    import torch
    case, bodies = _case(pkg, scene)
    p = case.sc.params
    spec = dict(wall=WALL, bodies=[BODY]) if scene == "body" else dict(wall=WALL)
    first = None
    for name in sorted(SD.PATHS):
        s, P, _, _ = _system(pkg, case, bodies, SD.PATHS[name])
        try:
            n = s.fluid.n
            groups = _np(s.body_local())[:, 3].astype(np.int64) if bodies else None
            beta = [WALL] + ([BODY] if scene == "body" else [])
            pos = s.state()["pos"]
            off = _off_grid(s, pos)
            ref, lo, hi = AR.accel(P, beta, p.rho0, p.rho_boundary, groups, AR.distance_error(pos), off)
            out = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
            s.adhesion_accel(out, spec)
            got = _np(out)
            ref64.assert_per_element(got, ref, ref64.TAU, f"{scene}/{name} a_i")
            st = s.adhesion_stats()
            assert lo <= st["wetted"] <= hi, (st["wetted"], lo, hi)
            if scene in ("walls", "body"):     # (config0's block lies more than R from every wall, and so does the body scene's)
                assert lo > 0, "no fluid particle in the band of a boundary particle"
            amax = np.sqrt((got.astype(np.float64) ** 2).sum(1)).max()
            assert abs(st["max_accel"] - amax) <= 1e-6 * amax, (st["max_accel"], amax)
            if scene == "body_without_entry":
                with_body, _, _ = AR.accel(P, [WALL, BODY], p.rho0, p.rho_boundary, groups, AR.distance_error(pos), off)
                assert np.abs(with_body.value - ref.value).max() > 1e-3 * np.abs(ref.value).max(), "the body touches no fluid"
            if first is None:
                first = bits(got)
            else:
                assert np.array_equal(bits(got), first), f"{scene}: path {name} differs from the first path"
        finally:
            s.close()


# ---- 2. momentum with a dynamic body ----------------------------------------------------------------------------------------
def _dynamic_plate(sc, mass):
    body = TIV._plate(sc.fluid.mean(0))
    body["mass"], body["inertia"] = mass, [1e-7, 1e-7, 1e-7]
    return body


@pytest.mark.parametrize("held", [False, True])
@pytest.mark.parametrize("moved", [False, True])
def test_reaction_balances_the_fluid(pkg, built, moved, held):
    """walls at 0, the plate at 90: one sphk_adhesion and sphk_bodies_integrate give sum m_i dv_i + J = 0 and the float64 {J, H};
    moved: the fluid advected by up to 0.6 cells after the search first, so that the reaction must reach two cells; held: the plate
    has M = 0 (a force sensor; a second, dynamic plate far from the fluid declares the dynamics) and reports the same J.  A call
    refused for a missing fluid mass changes nothing."""
    _gpu()
    import ctypes as C
    import torch
    from cpp_fluid_particles_b200 import capi
    from oracle import oracle as O
    case, _ = TIV._case(pkg, "body")
    p = case.sc.params
    bodies = [_dynamic_plate(case.sc, 0.0 if held else 1e-3)]
    if held:
        bodies.append(_dynamic_plate(case.sc, 1e-3))
        bodies[1]["position"] = [0.4, 0.4, 0.4]
    s, _, _, mass = _system(pkg, case, bodies)
    try:
        n = s.fluid.n
        if moved:
            rng = np.random.default_rng(11)
            v = (rng.uniform(-1.0, 1.0, (n, 3)) * (0.6 * p.cell_length / p.dt)).astype(F)
            s.fluid.vel[:n] = torch.from_numpy(v).cuda()
            s.refresh()
            s.advect()
            s.fluid.vel.zero_()
            s.refresh()
        st = s.state()
        g = O.grid(p.cell_size, p.cell_length, hash_rcp=s.device_rcp(p.cell_length))
        P = ref64.Pairs(O.SceneArrays(st["pos"], mass, st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius))
        v0 = _np(s.fluid.vel[:n]).astype(np.float64)
        spec = dict(wall=0.0, bodies=[BODY, 0.0] if held else [BODY])
        s.adhesion = spec
        live = s.scene_abi()
        bad = type(live).from_buffer_copy(live)      # (a copy: the system keeps its own scene)
        bad.fluid.mass = None
        assert s.L.sphk_adhesion(s.ctx, C.byref(bad), C.byref(capi.adhesion(spec)), C.c_float(s.dt), C.c_float(p.rho0),
                                 C.c_float(p.rho_boundary)) == -1
        assert np.array_equal(bits(_np(s.fluid.vel[:n])), bits(v0.astype(F))), "a refused call wrote velocities"
        s.adhesion_step()
        assert s.L.sphk_bodies_integrate(s.ctx, C.c_float(s.dt), (C.c_float * 3)(0.0, 0.0, 0.0)) == 0
        JH = s.body_impulse()[0].astype(np.float64)
        dp = (mass.astype(np.float64)[:, None] * (_np(s.fluid.vel[:n]) - v0)).sum(0)
        scale = (mass.astype(np.float64)[:, None] * np.abs(_np(s.fluid.vel[:n]) - v0)).sum(0).max()
        assert scale > 0, "the plate wets no fluid"
        assert np.abs(dp + JH[:3]).max() <= 1e-5 * scale, (dp, JH[:3])
        groups = _np(s.body_local())[:, 3].astype(np.int64)
        ref = AR.reaction(P, [0.0, BODY] + ([0.0] if held else []), p.rho0, p.rho_boundary, float(F(s.dt)), mass, st["posB"], groups,
                          s.body_pose()[:, :3])[0]
        assert np.abs(JH[:3] - ref[:3]).max() <= 1e-4 * np.abs(ref[:3]).max(), (JH[:3], ref[:3])
        assert np.abs(JH[3:] - ref[3:]).max() <= 1e-3 * np.abs(ref[3:]).max() + 1e-12, (JH[3:], ref[3:])
    finally:
        s.close()


# ---- 3. non-interference, graph, layers -------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_unused_changes_nothing(pkg, built, solver):
    """never set, set then cleared, and every beta 0: the same bits"""
    _gpu()
    a, b, c = _app(pkg, solver), _app(pkg, solver), _app(pkg, solver)
    b.set_adhesion(dict(wall=WALL)); b.set_adhesion(None)
    c.set_adhesion(dict(wall=0.0))
    try:
        for k in range(6):
            for x in (a, b, c):
                x.step()
            ra = a.download()
            _same(ra, b.download(), f"{solver} step {k} set then cleared")
            _same(ra, c.download(), f"{solver} step {k} beta 0")
    finally:
        for x in (a, b, c):
            x.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_graph_and_layers_agree(pkg, built, solver):
    """graph on and off give the same bits with adhesion on; the facade and the python engine agree bit for bit"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    from cpp_fluid_particles_b200 import capi
    sc = _wet_scene(pkg, solver)
    g, p = capi.SphApp(sc), capi.SphApp(sc)
    p.set_option(3, 0)
    e = engine.SphkSystem(sc)
    try:
        for x in (g, p):
            x.set_adhesion(dict(wall=WALL))
        e.adhesion = dict(wall=WALL)
        wetted = 0
        for k in range(8):
            g.step(); p.step(); e.step()
            rg = g.download()
            _same(rg, p.download(), f"{solver} step {k}: graph vs plain")
            _same(rg, e.state(), f"{solver} step {k}: facade vs engine", ("pos", "density"))
            wetted = max(wetted, g.adhesion_stats()["wetted"])
            assert g.adhesion_stats() == e.adhesion_stats()
        assert g.step_graph_active() and not p.step_graph_active()
        assert wetted > 0
    finally:
        g.close(); p.close(); e.close()


CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")


@pytest.mark.parametrize("solver", SOLVERS)
def test_headless_dump_agrees(pkg, built, solver, tmp_path):
    """the mini block lowered into the floor's band (origin y 0.0325: first layer 3R/4 above the shell): the headless app's dump, the
    facade and the python engine agree bit for bit with adhesion on, and adhesion changed the result"""
    _gpu()
    import dataclasses
    from cpp_fluid_particles_b200 import capi, engine
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    base = [CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--box", str(box), "--block", str(nx), str(ny), str(nz),
            "--origin", repr(float(origin[0])), "0.0325", repr(float(origin[2])), "--quiet"] + (["--iters", "4"] if solver != "wcsph" else [])
    prefix = str(tmp_path / "scene")
    r = subprocess.run(base + ["--emit-scene", prefix], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    sc = pkg.scene.benchmark_scene("mini", solver)
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(np.fromfile(prefix + ".fluid.f32", np.float32).reshape(-1, 3)))
    assert np.array_equal(np.fromfile(prefix + ".boundary.f32", np.float32).reshape(-1, 3), sc.boundary)
    dump = str(tmp_path / "dump")
    r = subprocess.run(base + ["--frames", "4", "--adhesion", repr(WALL), "--dump", dump], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    app, off = capi.SphApp(sc), capi.SphApp(sc)
    e = engine.SphkSystem(sc)
    try:
        app.set_adhesion(dict(wall=WALL))
        e.adhesion = dict(wall=WALL)
        for _ in range(4):
            app.step(); off.step(); e.step()
        a = app.download()
        _same(a, e.state(), f"{solver}: facade vs python engine")
        pos = np.fromfile(dump + ".pos.f32", np.float32).reshape(-1, 3)
        den = np.fromfile(dump + ".density.f32", np.float32)
        assert np.array_equal(bits(pos), bits(a["pos"])) and np.array_equal(bits(den), bits(a["density"])), "sph_headless"
        assert app.adhesion_stats()["wetted"] > 0
        assert not np.array_equal(bits(a["vel"]), bits(off.download()["vel"])), "adhesion must change the velocities"
    finally:
        app.close(); off.close(); e.close()


# ---- 4. physics -----------------------------------------------------------------------------------------------------------------
def _layer_scene(pkg, solver, layers=3):
    """the bottom `layers` lattice layers of the mini block, lowered so that the first starts 3R/4 above the floor's shell (in the
    band), under gravity reversed: +9.8 in y"""
    import dataclasses
    sc = pkg.scene.benchmark_scene("mini", solver)
    floor = sc.boundary[:, 1].min()
    fl = sc.fluid
    ys = np.unique(fl[:, 1])[:layers]
    fluid = fl[np.isin(fl[:, 1], ys)].copy()
    fluid[:, 1] += F(floor + 0.75 * sc.params.radius) - fluid[:, 1].min()
    params = dataclasses.replace(sc.params, gravity=(0.0, 9.8, 0.0))
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(fluid.astype(F)), params=params)


def _held(s, floor_tree, n1):
    """fraction of the first layer's count that lies within R of the floor's shell"""
    d, _ = floor_tree.query(s.state()["pos"], distance_upper_bound=s.p.radius)
    return np.isfinite(d).sum() / n1


# the balance beta of each scene from tests/adhesion_ref.py: g over the mean upward-opposing pull per unit beta on the first layer
@pytest.mark.parametrize("solver", SOLVERS)
def test_reversed_gravity_layer_hangs(pkg, built, solver):
    """a 3-layer film on the floor with gravity reversed, 0.2 s: at beta = 0 it leaves the floor (under 10 % of the first layer's
    count within R of the floor's shell); at 3x the balance beta the first layer stays within R (at least 90 %)"""
    _gpu()
    from scipy.spatial import cKDTree
    from cpp_fluid_particles_b200 import engine
    from oracle import oracle as O
    sc = _layer_scene(pkg, solver)
    p = sc.params
    floorB = sc.boundary[sc.boundary[:, 1] == sc.boundary[:, 1].min()]
    tree = cKDTree(floorB)
    n1 = int((sc.fluid[:, 1] == sc.fluid[:, 1].min()).sum())
    probe = engine.SphkSystem(sc, step0=False)
    try:
        probe.search_fluid()
        st = probe.state()
        g = O.grid(p.cell_size, p.cell_length, hash_rcp=probe.device_rcp(p.cell_length))
        P = ref64.Pairs(O.SceneArrays(st["pos"], st["mass"], st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius))
    finally:
        probe.close()
    unit, _, _ = AR.accel(P, [1.0], p.rho0, p.rho_boundary)
    first = st["pos"][:, 1] == st["pos"][:, 1].min()
    balance = 9.8 / np.mean(-unit.value[first, 1])
    steps = int(round(0.2 / p.dt))
    held = {}
    for k in (0.0, 1.0, 3.0, 10.0):
        s = engine.SphkSystem(sc)
        try:
            if k > 0:
                s.adhesion = dict(wall=k * balance)
            for _ in range(steps):
                s.step()
            assert np.isfinite(s.state()["pos"]).all()
            held[k] = _held(s, tree, n1)
        finally:
            s.close()
    print(f"\n{solver}: balance beta {balance:.1f}; first layer within R after {steps} steps: " +
          ", ".join(f"{k:g}x {v:.3f}" for k, v in held.items()))
    assert held[0.0] < 0.1
    assert held[3.0] >= 0.9
def _footprint(s):
    """fluid particles within R of a boundary particle"""
    from scipy.spatial import cKDTree
    st = s.state()
    d, _ = cKDTree(st["posB"]).query(st["pos"], distance_upper_bound=s.p.radius)
    return int(np.isfinite(d).sum())


# Not DFSPH: its density solve runs after the velocity stage and projects out the compression the pull causes.  The block's first
# layer, under the full column, is at rest density beyond the band, so it is pushed back out (footprint 968 with beta at 3x balance
# against 994 without, with the block's rebound).  An under-dense film is not: test_reversed_gravity_layer_hangs holds it on DFSPH too.
@pytest.mark.parametrize("solver", ["wcsph", "pbd"])
def test_settling_block_wets_more_walls(pkg, built, solver):
    """the mini block lowered into the band of the floor (_wet_scene) and left to settle: with beta at 3 times the value whose mean
    pull on the wetted particles balances g (the float64 reference on the initial state), more particles lie within R of the walls
    after 60 steps than without adhesion"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    from oracle import oracle as O
    sc = _wet_scene(pkg, solver)
    p = sc.params
    a, b = engine.SphkSystem(sc, step0=False), engine.SphkSystem(sc)
    try:
        a.search_fluid()
        st = a.state()
        g = O.grid(p.cell_size, p.cell_length, hash_rcp=a.device_rcp(p.cell_length))
        P = ref64.Pairs(O.SceneArrays(st["pos"], st["mass"], st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius))
        unit, _, _ = AR.accel(P, [1.0], p.rho0, p.rho_boundary)
        mag = np.sqrt((unit.value ** 2).sum(1))
        balance = 9.8 / np.mean(mag[mag > 0])
        a.close()
        a = engine.SphkSystem(sc)
        b.adhesion = dict(wall=3.0 * balance)
        for _ in range(60):
            a.step(); b.step()
        fa, fb = _footprint(a), _footprint(b)
        print(f"\n{solver}: balance beta {balance:.1f}; footprint {fa} without adhesion, {fb} with beta {3 * balance:.1f}")
        assert np.isfinite(b.state()["pos"]).all()
        assert fb > fa
    finally:
        a.close(); b.close()


# ---- 5. combinations ------------------------------------------------------------------------------------------------------------
def test_combinations_run_finite(pkg, built):
    """adhesion with heat, a rheology and CFL-adaptive steps in one system, and with an emitter and a sink in another"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "dfsph"))
    try:
        s.adhesion = dict(wall=WALL)
        s.thermal = dict(alpha=1e-3, beta=0.01, t_ref=20.0, wall=(60.0, 0.5))
        s.rheology = dict(model="cross", nu0=0.1, nu_inf=0.001, lam=1.0, m=1.0, nu_max=0.1)
        for _ in range(10):
            s.step()
        assert np.isfinite(s.state()["pos"]).all() and np.isfinite(s.state()["vel"]).all()
    finally:
        s.close()
    for extra in (["--cfl", "0.4", "--heat", "1e-3,0.01,20"], ["--tap", "2.5", "--drain", "0.2"]):
        r = _headless(["--solver", "dfsph", "--iters", "4", "--frames", "6", "--adhesion", "150"] + extra)
        assert np.isfinite(r["avg_ms_per_frame"]) and r["adhesion_wetted"] >= 0 and np.isfinite(r["adhesion_max_accel"]), r


# ---- 6. headless ------------------------------------------------------------------------------------------------------------------
def _wet_scene(pkg, solver):
    """the mini benchmark scene with its block lowered so that the bottom layer starts at 3R/4 above the floor's shell: in the band.
    (At rest the fluid of the shipped scenes stays about 1.24 R from the shell, beyond the band.)"""
    import dataclasses
    sc = pkg.scene.benchmark_scene("mini", solver)
    floor = sc.boundary[:, 1].min()
    fluid = sc.fluid.copy()
    fluid[:, 1] += F(floor + 0.75 * sc.params.radius) - fluid[:, 1].min()
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(fluid.astype(F)))


def _headless(args):
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--quiet"] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("solver", ["sph", "dfsph", "pbd"])
def test_headless_runs(built, solver):
    """--adhesion runs for every solver and reports its statistics; beta 0 wets nothing, beta 150 leaves a wetted film after the
    DFSPH and PBD dam-break waves"""
    _gpu()
    base = ["--solver", solver, "--frames", "60"] + (["--iters", "4"] if solver != "sph" else [])
    off = _headless(base + ["--adhesion", "0"])
    on = _headless(base + ["--adhesion", "150"])
    print(f"\n{solver}: wetted {off['adhesion_wetted']} at beta 0, {on['adhesion_wetted']} at beta 150, max accel "
          f"{on['adhesion_max_accel']}")
    assert off["adhesion_wetted"] == 0 and off["adhesion_max_accel"] == 0.0
    assert np.isfinite(on["adhesion_max_accel"])
    if solver != "sph":         # (the WCSPH wave, at dt = 1 ms, reaches no wall's band in these 60 ms)
        assert on["adhesion_wetted"] > off["adhesion_wetted"]


def test_headless_floating_cube_feels_adhesion(built):
    """--float: BODYBETA > 0 changes the cube's impulse and position"""
    _gpu()
    base = ["--solver", "dfsph", "--iters", "4", "--frames", "30", "--float", "0.5"]
    a = _headless(base + ["--adhesion", "150,0"])
    b = _headless(base + ["--adhesion", "150,150"])
    assert a["body_impulse"] != b["body_impulse"] and a["body_position"] != b["body_position"], (a, b)
