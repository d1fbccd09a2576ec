"""Probes and water-level gauges on the GPU: records and levels per element against the float64 reference (tests/probe_ref.py) on
every execution path and in states whose positions moved since the search, the lattice against the point entry bit for bit, zero
interference with the particles (plain steps and graph replay), the recorded series (graph replay, on-demand samples, the ring's
wrap, CFL times, an open system), the layers (headless CSV, facade, python engine), physics that holds by construction, and the
refusals."""
import os
import subprocess

import numpy as np
import pytest

import probe_ref as PR
import sweep_driver as SD
import test_gpu_implicit_viscosity as TIV
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
_gpu, _np, _same = TIV._gpu, TIV._np, TIV._same
# absolute allowance beyond tau * mag: the float32 rounding of rho(x) = sum m W / S and of the velocity quotients is relative to the
# result (covered by mag); the floor only absorbs the last-ulp rounding of values that cancel to ~0 (a velocity component near 0)
FLOOR = 1e-9


def _in_grid(p, pts):
    c = np.trunc(np.asarray(pts, np.float64) / np.float64(F(p.cell_length)))
    return np.all((c >= 0) & (c < np.asarray(p.cell_size)[None, :]), 1)


def _points(p, pos, rng):
    """inside the fluid, on particles (r = 0), on exact cell faces, outside the grid, and where no fluid is within reach"""
    inside = pos[rng.choice(len(pos), 1000, replace=False)] + rng.uniform(-0.5, 0.5, (1000, 3)).astype(F) * F(p.radius)
    on = pos[rng.choice(len(pos), 50, replace=False)]
    cl = F(p.cell_length)
    faces = (np.round(pos[rng.choice(len(pos), 50, replace=False)] / cl) * cl).astype(F)
    outside = np.array([[-1.0, 0.1, 0.1], [0.1, 5.0, 0.1], [0.1, 0.1, -0.3]], F)
    dry = np.array([[0.5 * p.space[0], 0.97 * p.space[1], 0.5 * p.space[2]], [0.02, 0.9 * p.space[1], 0.02]], F)
    return np.ascontiguousarray(np.concatenate([inside, on, faces, outside, dry]).astype(F))


def _check_records(got, pts, st, p, pressure=None, temperature=None):
    counted = np.arange(len(st["pos"])) < int(st["cell_start"][-1])
    ref, mag, lo, hi = PR.records(pts, st["pos"], st["vel"], st["mass"], st["density"], p.radius, counted, ~_in_grid(p, pts),
                                  pressure, temperature)
    n = got[:, 7]
    assert np.all((n >= lo) & (n <= hi)), "n outside the rounding band at R"
    for c in range(7):
        if c in (5, 6) and np.isnan(ref[:, c]).all():
            assert np.isnan(got[:, c]).all(), f"field {c} must be NaN"
            continue
        err = np.abs(got[:, c].astype(np.float64) - ref[:, c])
        bound = PR.TAU * mag[:, c] + FLOOR
        assert np.all(err <= bound), f"field {c}: worst ratio {float(np.max(err / bound)):.3g} at {int(np.argmax(err / bound))}"
    return float(np.max(np.abs(got[:, 0] - ref[:, 0]) / np.maximum(mag[:, 0], 1e-30)))


def _system(pkg, scene, path):
    case, bodies = (TIV._case(pkg, "body") if scene == "body" else (SD.make_case(pkg, scene), None))
    s, _, _, _ = TIV._system(pkg, case, bodies, path)
    return s, case.sc.params


# ---- 1. records and levels per element ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["config0", "config0_mass", "walls", "body"])
@pytest.mark.parametrize("state", ["searched", "advected"])
def test_records_per_element_on_every_path(pkg, built, scene, state):
    """records against float64 at points inside the fluid, on particles, on cell faces, outside the grid and in dry air; after an
    advect the cell ranges are stale (reach 2); the same bits on every path (the probe walk ignores the list)"""
    _gpu()
    import torch
    first = None
    for name in sorted(SD.PATHS):
        s, p = _system(pkg, scene, SD.PATHS[name])
        try:
            s.density()
            s.pressure()
            if state == "advected":
                # up to half a cell in one advect: pairs within R whose particle is listed two rows from the point's cell
                s.fluid.vel.add_(torch.tensor([[2.7, -5.1, 1.8]], device=s.device))
                s.refresh()                     # the records carry the velocities sphk_advect reads
                s.advect()
            st = s.state()
            pts = _points(p, st["pos"][: int(st["cell_start"][-1])], np.random.default_rng(7))
            got = _np(s.probe_sample(torch.from_numpy(pts).to(s.device)))
            _check_records(got, pts, st, p, pressure=st["pressure"] if s._probe_sources()[0] is not None else None)
            assert np.all(got[-5:-2, 7] == 0), "outside the grid"
            if first is None:
                first = got
            else:
                assert np.array_equal(bits(got), bits(first)), f"path {name} differs"
        finally:
            s.close()


def test_records_after_a_pbd_step(pkg, built):
    """the state a PBD step leaves (positions moved by the corrections and the prediction): reach 2"""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "pbd"))
    try:
        for _ in range(3):
            s.step()
        p = s.p
        st = s.state()
        pts = _points(p, st["pos"], np.random.default_rng(3))
        got = _np(s.probe_sample(torch.from_numpy(pts).to(s.device)))
        _check_records(got, pts, st, p)
        assert np.isnan(got[:, 5]).all() and np.isnan(got[:, 6]).all()
    finally:
        s.close()


def _field(pos, seed):
    """a non-uniform per-particle field: linear in position plus noise, so a wrong index or normalisation shows"""
    rng = np.random.default_rng(seed)
    return (20.0 + 30.0 * pos[:, 0] - 12.0 * pos[:, 1] + rng.uniform(-1.0, 1.0, len(pos))).astype(F)


def test_pressure_and_temperature_per_element(pkg, built):
    """p of a WCSPH state and T with heat transfer on, per element against float64, in the python engine and through the class
    layer (the facade passes the solver's pressure array and temperatureField()).  The WCSPH column of the hydrostatic test, after
    100 steps: the mini dam-break's block has p = 0 everywhere (its densities lie below rho0, and the equation of state clamps)."""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    sc, _ = _column(pkg, "wcsph")
    spec = dict(alpha=1e-4, beta=0.0, t_ref=20.0)
    s, a = engine.SphkSystem(sc), capi.SphApp(sc)
    try:
        s.thermal = spec
        a.set_thermal(spec)
        for _ in range(100):
            s.step(); a.step()
        p = s.p
        # the python engine: its pressure and its temperature tensor
        n = s.fluid.n
        s.temperature[:n] = torch.from_numpy(_field(s.state()["pos"], 1)).to(s.device)
        st = s.state()
        T = _np(s.temperature[:n])
        pts = _points(p, st["pos"][: int(st["cell_start"][-1])], np.random.default_rng(5))
        got = _np(s.probe_sample(torch.from_numpy(pts).to(s.device)))
        assert np.any(got[:, 5] > 0) and np.all(np.isfinite(got[:, 5:7]))
        _check_records(got, pts, st, p, pressure=st["pressure"], temperature=T)
        # the class layer (every particle of the mini tank is in the grid)
        d = a.download()
        a.upload_temperature(_field(d["pos"], 2))
        T = a.download_temperature()
        got = a.sample_probes(pts)
        st = dict(d, cell_start=np.array([len(d["pos"])]))
        assert np.any(got[:, 5] > 0)
        _check_records(got, pts, st, p, pressure=d["pressure"], temperature=T)
    finally:
        s.close(); a.close()


def test_reach_two_after_a_move(pkg, built):
    """the reach contract: after a move of less than a cell since the search, a particle listed two cell rows from the probe's cell
    (it sat near the low face of its cell and moved 0.7 of a cell towards the probe) is within R and must count"""
    _gpu()
    import torch
    s, p = _system(pkg, "config0", SD.PATHS["list"])
    try:
        s.density()
        st = s.state()
        L = float(F(p.cell_length))
        live = int(st["cell_start"][-1])
        frac = st["pos"][:live, 0] / L - np.floor(st["pos"][:live, 0] / L)
        cand = np.nonzero((frac > 0.02) & (frac < 0.15) & (st["pos"][:live, 0] > 3 * L))[0][:16]
        assert cand.size >= 8
        pts, moves = [], np.zeros((s.fluid.n, 3), F)
        for j in cand[:1]:
            cj = np.floor(st["pos"][j, 0] / L)
            x = F((cj - 1) * L - 0.05 * L)                               # two cell rows below the particle's cell
            pts.append([x, st["pos"][j, 1], st["pos"][j, 2]])
            moves[j, 0] = (x + F(0.5 * p.radius) - st["pos"][j, 0]) / F(s.dt)
        s.fluid.vel.copy_(torch.from_numpy(moves).to(s.device))
        s.refresh()
        s.advect()
        assert abs(float(s.state()["pos"][cand[0], 0]) - float(pts[0][0] + F(0.5 * p.radius))) < 1e-5
        st = s.state()
        pts = np.asarray(pts, F)
        got = _np(s.probe_sample(torch.from_numpy(pts).to(s.device)))
        _check_records(got, pts, st, p)
    finally:
        s.close()


def test_gauge_levels_per_element(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "dfsph"))
    try:
        for _ in range(3):
            s.step()
        p, st = s.p, s.state()
        top = 0.9 * p.space[1]
        xs = np.linspace(0.12, 0.38, 12)
        gauges = [((float(x), top, float(z), 128 if k % 2 else 64)) for k, (x, z) in enumerate(zip(xs, xs[::-1]))]
        gauges = [((g[0], 0.002, g[2]), (g[0], g[1], g[2]), g[3]) for g in gauges]      # upwards, along -G
        gauges.append(((0.45, 0.8 * p.space[1], 0.45), (0.45, top, 0.45), 8))          # dry
        got = _np(s.gauge_levels(gauges, 0.5))
        counted = np.arange(len(st["pos"])) < int(st["cell_start"][-1])
        ref = PR.gauge_levels(gauges, 0.5, st["pos"], st["mass"], st["density"], p.radius, counted, lambda q: ~_in_grid(p, q))
        checked = 0
        for g, (lv, bound, amb) in zip(got, ref):
            if amb:
                continue
            assert abs(float(g) - lv) <= bound, (g, lv, bound)
            checked += 1
        assert checked >= 8 and got[-1] == -1.0
        assert np.count_nonzero(got[:-1] > 0) >= 6
    finally:
        s.close()


# ---- 2. the lattice -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [(1, 1, 1), (7, 1, 1), (1, 1, 9), (5, 6, 7), (128, 128, 128)])
def test_lattice_equals_points(pkg, built, dims):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "wcsph"))
    try:
        s.step()
        origin, spacing = (F(0.143), F(0.0571), F(0.151)), F(0.5 * s.p.space[0] / 128.0 * 2.0)
        lat = s.probe_lattice(origin, float(spacing), dims)
        i, j, k = np.meshgrid(*[np.arange(d, dtype=F) for d in dims], indexing="ij")
        pts = np.stack([F(origin[0]) + spacing * i, F(origin[1]) + spacing * j, F(origin[2]) + spacing * k], -1).astype(F).reshape(-1, 3)
        got = s.probe_sample(torch.from_numpy(np.ascontiguousarray(pts)).to(s.device))
        assert torch.equal(lat.reshape(-1, 8).view(torch.int32), got.view(torch.int32))
        assert int((lat[..., 7] > 0).sum()) > 0 or int(np.prod(dims)) < 10
    finally:
        s.close()


# ---- 3. zero interference and the series ---------------------------------------------------------------------------------------
PROBES = [[0.2, 0.06, 0.2], [0.25, 0.1, 0.22], [0.3, 0.2, 0.3], [0.45, 0.45, 0.45]]
GAUGES = [((0.2, 0.002, 0.2), (0.2, 0.4, 0.2), 96), ((0.35, 0.002, 0.3), (0.35, 0.4, 0.3), 64)]     # upwards, along -G


def _app(pkg, solver, graph=True):
    from cpp_fluid_particles_b200 import capi
    a = capi.SphApp(pkg.scene.benchmark_scene("mini", solver))
    if not graph:
        a.set_option(3, 0)
    return a


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_interference_and_graph_series(pkg, built, solver):
    """probes on and off give the same particles, plain and replayed; the replayed series equals the plain one bit for bit, and
    every row equals an on-demand sample taken after its step"""
    _gpu()
    off, on, plain = _app(pkg, solver), _app(pkg, solver), _app(pkg, solver, graph=False)
    try:
        on.set_probes(PROBES, GAUGES, capacity=16)
        plain.set_probes(PROBES, GAUGES, capacity=16)
        samples = []
        for k in range(8):
            for a in (off, on, plain):
                a.step()
            samples.append(plain.sample_probes(PROBES))
            ref = off.download()
            _same(ref, on.download(), f"{solver} step {k}: probes on", ("pos", "vel", "density", "pressure"))
            _same(ref, plain.download(), f"{solver} step {k}: probes on, no graph", ("pos", "vel", "density", "pressure"))
        assert on.step_graph_active() and not plain.step_graph_active()
        a, b = on.probe_series(), plain.probe_series()
        assert a["records"].shape == (8, 4, 8) and a["levels"].shape == (8, 2) and a["overwritten"] == 0
        assert np.array_equal(a["steps"], np.arange(1, 9)) and np.array_equal(a["steps"], b["steps"])
        assert np.array_equal(bits(a["records"]), bits(b["records"])) and np.array_equal(bits(a["levels"]), bits(b["levels"]))
        assert np.array_equal(bits(a["records"]), bits(np.stack(samples)))
        assert np.all(a["records"][:, 0, 7] > 0) and np.all(a["records"][:, 3, 7] == 0)
        assert np.isnan(a["records"][:, :, 5]).all() == (solver != "wcsph")
        assert np.allclose(a["times"], np.arange(1, 9) * np.float64(F(pkg.scene.benchmark_scene("mini", solver).params.dt)) +
                           np.float64(F(pkg.scene.benchmark_scene("mini", solver).params.dt)), rtol=1e-12)
    finally:
        off.close(); on.close(); plain.close()


def test_ring_wraps(pkg, built):
    _gpu()
    a = _app(pkg, "dfsph")
    try:
        a.set_probes(PROBES, GAUGES, capacity=5)
        for _ in range(8):
            a.step()
        s = a.probe_series()
        assert s["overwritten"] == 3 and np.array_equal(s["steps"], np.arange(4, 9)) and s["records"].shape[0] == 5
        last = a.sample_probes(PROBES)
        assert np.array_equal(bits(s["records"][-1]), bits(last))
        a.set_probes([], [])                      # off: no rows any more
        a.step()
        with pytest.raises(RuntimeError):
            a.set_probes(PROBES, GAUGES, capacity=0)
    finally:
        a.close()


def test_cfl_series_carries_the_simulated_time(pkg, built):
    _gpu()
    a = _app(pkg, "dfsph")
    try:
        a.set_adaptive_dt(0.4)
        a.set_probes(PROBES, GAUGES, capacity=256)
        k1, _ = a.advance(0.02)
        k2, _ = a.advance(0.02)
        s = a.probe_series()
        assert len(s["steps"]) == k1 + k2 and np.all(np.diff(s["times"]) > 0)
        assert s["times"][-1] == a.adaptive_stats()["simulated_time"]
    finally:
        a.close()


def test_open_system_gauge_under_the_tap_rises(pkg, built):
    """a tap into the mini tank: the gauge under it ends higher than in the same tank without the tap, and higher than it started"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    em = {"origin": (0.25, 0.40, 0.25), "direction": (0.0, -1.0, 0.0), "speed": 1.0, "spacing": 0.02, "width": 5, "height": 4}
    tap = capi.SphApp(sc, max_fluid=3 * len(sc.fluid), emitters=[em], sinks=[])
    closed = capi.SphApp(sc, max_fluid=3 * len(sc.fluid), emitters=[], sinks=[])
    gauge = [((0.25, 0.002, 0.25), (0.25, 0.45, 0.25), 128)]
    try:
        for a in (tap, closed):
            a.set_probes([], gauge, capacity=400)
            for _ in range(400):
                a.step()
        lt, lc = tap.probe_series()["levels"][:, 0], closed.probe_series()["levels"][:, 0]
        assert tap.fluid_count > len(sc.fluid) + 500
        assert lt[-1] > lc[-1] + 0.005 and lt[-1] > lt[200], (lt[200], lt[-1], lc[-1])
    finally:
        tap.close(); closed.close()


# ---- 4. the layers agree -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_layers_agree(pkg, built, solver, tmp_path):
    """the headless --probe-out CSV, the facade's series and the python engine's series, bit for bit"""
    _gpu()
    import dataclasses
    from cpp_fluid_particles_b200 import capi, engine
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    base = [CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--box", str(box), "--block", str(nx), str(ny), str(nz),
            "--origin", *[repr(float(o)) for o in origin], "--quiet"] + (["--iters", "4"] if solver != "wcsph" else [])
    prefix = str(tmp_path / "scene")
    r = subprocess.run(base + ["--emit-scene", prefix], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    sc = pkg.scene.benchmark_scene("mini", solver)
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(np.fromfile(prefix + ".fluid.f32", np.float32).reshape(-1, 3)))
    csv = str(tmp_path / "probes.csv")
    args = []
    for q in PROBES:
        args += ["--probe", ",".join(repr(float(x)) for x in q)]
    for a_, b_, k in GAUGES:
        args += ["--gauge", ",".join(repr(float(x)) for x in (*a_, *b_, k))]
    r = subprocess.run(base + ["--frames", "5", "--probe-out", csv] + args, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    rows = np.loadtxt(csv, delimiter=",", skiprows=1, ndmin=2)
    app, e = capi.SphApp(sc), engine.SphkSystem(sc)
    try:
        app.set_probes(PROBES, GAUGES)
        e.set_probes(PROBES, GAUGES)
        for _ in range(5):
            app.step(); e.step()
        a, b = app.probe_series(), e.probe_series()
        for k in ("records", "levels"):
            assert np.array_equal(bits(a[k]), bits(b[k])), f"{solver}: facade vs python engine {k}"
        assert np.array_equal(a["steps"], b["steps"]) and np.array_equal(a["times"], b["times"])
        assert np.array_equal(rows[:, 0].astype(np.int64), a["steps"]) and np.array_equal(rows[:, 1], a["times"])
        flat = np.concatenate([a["records"].reshape(5, -1), a["levels"]], 1).astype(np.float32)
        csv32 = rows[:, 2:].astype(np.float32)
        assert np.array_equal(np.isnan(csv32), np.isnan(flat)), f"{solver}: headless CSV NaNs"
        assert np.array_equal(bits(np.nan_to_num(csv32)), bits(np.nan_to_num(flat))), f"{solver}: headless CSV"
    finally:
        app.close(); e.close()


# ---- 5. physics -------------------------------------------------------------------------------------------------------------------
def test_dam_break_gauges_wet_in_order(pkg, built, tmp_path):
    """the mini dam-break: gauges at increasing distance from the block wet in that order, and the level at the block falls"""
    _gpu()
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    csv = str(tmp_path / "dam.csv")
    xs = [0.2, 0.3, 0.38, 0.46]
    args = []
    for x in xs:
        args += ["--gauge", f"{x},0.002,0.25,{x},0.4,0.25,128"]
    r = subprocess.run([CLI, "--solver", "dfsph", "--box", str(box), "--block", str(nx), str(ny), str(nz), "--origin",
                        *[repr(float(o)) for o in origin], "--quiet", "--frames", "150", "--probe-out", csv] + args,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lv = np.loadtxt(csv, delimiter=",", skiprows=1, ndmin=2)[:, 2:]
    wet = [int(np.argmax(lv[:, g] > 0)) if np.any(lv[:, g] > 0) else len(lv) for g in range(lv.shape[1])]
    assert wet[1] <= wet[2] <= wet[3] and wet[3] < len(lv), wet
    assert lv[-1, 0] < lv[0, 0] - 0.02, (lv[0, 0], lv[-1, 0])


def _column(pkg, solver, layers=8):
    """a fluid column filling the mini tank's floor: 23 x layers x 23 particles at the fluid spacing from 0.025 (the first layer
    one spacing above the floor's shell), so it has nowhere to flow"""
    import dataclasses
    sc = pkg.scene.benchmark_scene("mini", solver)
    g = (F(0.025) + F(0.02) * np.arange(23, dtype=F)).astype(F)
    y = (F(0.025) + F(0.02) * np.arange(layers, dtype=F)).astype(F)
    fl = np.stack(np.meshgrid(g, y, g, indexing="ij"), -1).reshape(-1, 3)[:, [0, 1, 2]].astype(F)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(fl)), float(y[-1] + F(0.01))


COLUMN_XZ = [(0.15, 0.15), (0.25, 0.25), (0.35, 0.2), (0.2, 0.35), (0.3, 0.3)]
# measured once on an NVIDIA H100 80GB HBM3 (DESIGN.md section 2.13) and set with the margins stated there
COLUMN_LEVEL_TOL = 0.02          # one fluid spacing: the issue's bound
COLUMN_SPEED_MAX = 0.05
HYDROSTATIC_SLOPE_TOL = 0.35


def test_dfsph_column_at_rest(pkg, built):
    """a DFSPH column at rest: its gauges stay within one spacing of the surface derived from the particle lattice (the highest
    particle near the gauge plus half the settled layer spacing: the column first sags until its densities reach rho0), and the
    interior is still"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc, _ = _column(pkg, "dfsph")
    s = engine.SphkSystem(sc)
    try:
        interior = [(x, y, z) for x, z in COLUMN_XZ for y in (0.06, 0.09, 0.12)]
        s.set_probes(interior, [((x, 0.002, z), (x, 0.4, z), 256) for x, z in COLUMN_XZ], capacity=400)
        for _ in range(300):
            s.step()
        ser = s.probe_series()
        pos = s.state()["pos"].astype(np.float64)
        layer = (pos[:, 1].max() - pos[:, 1].min()) / 7.0
        surf = []
        for x, z in COLUMN_XZ:
            near = np.hypot(pos[:, 0] - x, pos[:, 2] - z) <= 0.02
            surf.append(pos[near, 1].max() + 0.5 * layer - 0.002)
        lv, rec = ser["levels"][-100:], ser["records"][-100:]
        speed = np.sqrt((rec[:, :, 2:5].astype(np.float64) ** 2).sum(-1))
        err = np.abs(lv - np.array(surf)[None, :])
        print(f"MEASURED dfsph column: layer {layer:.5f} m, surface {np.round(surf, 4).tolist()}, level error {err.max():.5f} m, "
              f"max interior |v| {speed.max():.5f} m/s")
        assert np.all(err <= COLUMN_LEVEL_TOL)
        assert speed.max() <= COLUMN_SPEED_MAX
    finally:
        s.close()


def test_wcsph_hydrostatic_pressure(pkg, built):
    """a settled WCSPH column: the interpolated p rises monotonically with depth along vertical lines; its slope is the slope of the
    particles' own pressures, and within HYDROSTATIC_SLOPE_TOL of rho0 |g| (time mean over the last 200 recorded steps).  The
    particles themselves settle about 26 % below rho0 |g| (DESIGN.md section 2.13): that is the solver's discrete equilibrium."""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc, _ = _column(pkg, "wcsph")
    s = engine.SphkSystem(sc)
    p = s.p
    ys = np.arange(0.065, 0.1151, 0.01)            # more than R from the floor's first fluid layer and from the surface
    try:
        s.set_probes([(x, y, z) for x, z in COLUMN_XZ for y in ys], [], capacity=200)
        for _ in range(3000):
            s.step()
        rec = s.probe_series()["records"][:, :, 5].astype(np.float64).reshape(-1, len(COLUMN_XZ), len(ys))
        pr = rec.mean(0)
        want = float(p.rho0) * abs(float(p.gravity[1]))
        slopes = np.array([-np.polyfit(ys, line, 1)[0] for line in pr])
        last = np.array([-np.polyfit(ys, line, 1)[0] for line in rec[-1]]).mean()
        st = s.state()
        x, pp = st["pos"].astype(np.float64), st["pressure"].astype(np.float64)
        inner = (x[:, 1] >= ys[0]) & (x[:, 1] <= ys[-1]) & np.all((x[:, [0, 2]] >= 0.1) & (x[:, [0, 2]] <= 0.4), 1)
        particles = -np.polyfit(x[inner, 1], pp[inner], 1)[0]
        err = np.abs(slopes / want - 1.0)
        print(f"MEASURED wcsph hydrostatic: probe slopes {np.round(slopes, 4).tolist()} (last step {last:.4f}), particles {particles:.4f}, "
              f"rho0|g| {want:.4f}, relative error max {err.max():.4f}")
        assert np.all(np.diff(pr, axis=1) < 0), "p must rise with depth"
        assert abs(last / particles - 1.0) <= 0.10, "the interpolated slope must be the particles' slope"
        assert err.max() <= HYDROSTATIC_SLOPE_TOL
    finally:
        s.close()


# ---- 6. refusals ---------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(pkg, built):
    _gpu()
    import ctypes as C
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    s = engine.SphkSystem(pkg.scene.benchmark_scene("mini", "dfsph"))
    try:
        s.set_probes(PROBES, GAUGES, capacity=4)
        for _ in range(2):
            s.step()
        before = s.probe_series()
        L, dev = s.L, s.device
        out = torch.full((4, 8), 7.0, device=dev)
        bad_pts = torch.tensor([[0.1, float("nan"), 0.1]] * 4, device=dev)
        assert L.sphk_probe_sample(s.ctx, s._s(), engine._ptr(bad_pts), C.c_int(4), None, None, engine._ptr(out)) == -1
        assert L.sphk_probe_sample(s.ctx, s._s(), engine._ptr(out), C.c_int(4), None, None, engine._ptr(out)) == -1   # aliased input
        assert L.sphk_probe_sample(s.ctx, s._s(), engine._ptr(out), C.c_int(1), None, None, engine._ptr(s.fluid.density)) == -1
        for spacing, dims in ((0.0, (2, 2, 2)), (float("nan"), (2, 2, 2)), (0.01, (0, 2, 2)), (0.01, (65536, 65536, 2))):
            assert L.sphk_probe_lattice(s.ctx, s._s(), (C.c_float * 3)(0.1, 0.1, 0.1), C.c_float(spacing), (C.c_int * 3)(*dims), None,
                                        None, engine._ptr(out)) == -1
        g, n = capi.gauge_structs(GAUGES, 0.5)
        for th in (0.0, -1.0, float("nan")):
            assert L.sphk_gauge_levels(s.ctx, s._s(), g, C.c_int(n), C.c_float(th), engine._ptr(out)) == -1
        assert L.sphk_gauge_levels(s.ctx, s._s(), g, C.c_int(capi.GAUGE_LIMIT + 1), C.c_float(0.5), engine._ptr(out)) == -1
        assert torch.all(out == 7.0)
        with pytest.raises(ValueError):
            s.set_probes(np.zeros((capi.PROBE_LIMIT + 1, 3)) + 0.1)
        with pytest.raises(ValueError):
            s.set_probes([], GAUGES * 33)
        for cap in (0, capi.PROBE_CAPACITY_LIMIT + 1):
            with pytest.raises(ValueError):
                s.set_probes(PROBES, GAUGES, capacity=cap)
        after = s.probe_series()
        for k in ("records", "levels", "steps"):
            assert np.array_equal(bits(before[k]), bits(after[k]))
        assert after["overwritten"] == before["overwritten"]
        assert s.set_probes(np.zeros((capi.PROBE_LIMIT, 3)) + 0.1, GAUGES * 32, capacity=2) is None    # the caps themselves are fine
        assert s.set_probes(PROBES, GAUGES, capacity=capi.PROBE_CAPACITY_LIMIT) is None
    finally:
        s.close()


# ---- 7. the headless app with probes under blocking launches (compute-sanitizer with SPHK_SANITIZER=1) ----------------------------
def test_headless_with_probes_runs_clean(built, tmp_path):
    import shutil
    csv = str(tmp_path / "p.csv")
    cmd = [CLI, "--solver", "pbd", "--frames", "3", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055", "0.135",
           "--quiet", "--iters", "2", "--probe", "0.2,0.1,0.2", "--probe", "0.2,0.2,0.2", "--gauge", "0.2,0.002,0.2,0.2,0.4,0.2,200",
           "--probe-out", csv]
    env = dict(os.environ, SPHK_STEP_GRAPH="0", CUDA_LAUNCH_BLOCKING="1")
    if os.environ.get("SPHK_SANITIZER") == "1":
        exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
        cmd = [exe, "--tool", "memcheck", "--error-exitcode", "9"] + cmd
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stdout[-4000:]
    assert "error" not in r.stdout.lower().replace("error summary: 0 errors", ""), r.stdout[-4000:]
    rows = np.loadtxt(csv, delimiter=",", skiprows=1, ndmin=2)
    assert rows.shape == (3, 2 + 16 + 1) and np.isfinite(rows[:, [2, 3, 4, 5, 6, 9]]).all()
