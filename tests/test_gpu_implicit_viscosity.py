"""Implicit viscosity on the GPU: the two sweeps of the solve per element on every execution path against the float64
reference (tests/implicit_visc_ref.py), the whole solve against the exact float64 solution and the float64 PCG, momentum and
energy, a fluid at rest, off means off, the step graph, the four layers (class layer, facade, python engine, sph_headless),
argument validation, and the physics of a viscous dam break and a stirred tank."""
import dataclasses
import os
import shutil
import subprocess

import numpy as np
import pytest

import implicit_visc_ref as IV
import ref64
import sweep_driver as SD
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
NU, NU_B = 0.05, 0.03
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
NU_CRIT_MINI = 0.011992        # tests/test_cpu_implicit_viscosity.py: the explicit limit on the mini DFSPH scene
WORK_D = 64 + 6 * 1024         # float offset of D in the solve's workspace (state head + double partials)


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _np(t):
    return t.detach().cpu().numpy().copy()


def _plate(centre, v=(0.3, 0.0, -0.2), w=(0.0, 4.0, 0.0), sb=0.0198):
    """a moving plate (kinematic body) of boundary-lattice spacing through the middle of the mini block"""
    g = (np.arange(-3, 4) * sb).astype(F)
    x, y = np.meshgrid(g, g, indexing="ij")
    pts = np.stack([x.ravel(), y.ravel(), np.zeros(x.size, F)], 1).astype(F)
    return {"points": pts, "position": [float(c) for c in centre], "orientation": [0.0, 0.0, 0.0, 1.0],
            "linear_velocity": list(v), "angular_velocity": list(w)}


SCENES = ["config0", "config0_mass", "walls", "n1", "n31", "n33", "body"]


def _oblique(sc):
    """the plate of _plate turned 0.9 rad about (1, 1, 0): its boundary terms make D_i anisotropic off the axes.  Fluid lattice
    points closer than half a boundary spacing to it are dropped."""
    c = sc.fluid.mean(0).astype(np.float64)
    a = np.array([1.0, 1.0, 0.0]) / np.sqrt(2.0)
    q = np.r_[a * np.sin(0.45), np.cos(0.45)]
    body = dict(_plate(c), orientation=[float(x) for x in q])
    x, y, z, w = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    xp = c + body["points"].astype(np.float64) @ R.T
    keep = np.min(np.linalg.norm(sc.fluid[:, None].astype(np.float64) - xp[None], axis=2), 1) > 0.5 * 0.0198
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(sc.fluid[keep])), body


def _case(pkg, name):
    if name in ("body", "wide", "oblique"):
        sc = pkg.scene.make_scene("mini", solver="dfsph", jitter=0.004, max_iter=4, den_thr=-1.0, div_thr=-1.0)
        if name == "wide":          # masses log-uniform over a factor 49: the mass inner product matters
            return SD.Case(name, sc, mass="wide", lattice_like=False), None
        if name == "oblique":
            sc, body = _oblique(sc)
            return SD.Case(name, sc, mass="random", lattice_like=False), [body]
        return SD.Case(name, sc, mass="random", lattice_like=False), [_plate(sc.fluid.mean(0))]
    return SD.make_case(pkg, name), None


def _masses(case, n, m0):
    if case.mass == "wide":
        return (m0 * np.exp(np.random.default_rng(17).uniform(np.log(1 / 7), np.log(7), n))).astype(F)
    return SD.case_masses(case, n, m0)


def _system(pkg, case, bodies, path=SD.PATHS["list"]):
    """engine system on `path` with the case's masses; (system, float64 pairs, boundary velocities of the records)"""
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    from oracle import oracle as O
    s = engine.SphkSystem(case.sc, step0=False, use_list=path.use_list, list_capacity=path.kmax, bodies=bodies)
    p = case.sc.params
    s.set_option(capi.OPT_STAGED_LIST_BUILD, path.staged)
    s.set_option(capi.OPT_TILE, path.tile)
    s.set_use_list(path.use_list, path.skin)
    mass = _masses(case, s.fluid.n, p.m0)
    s.fluid.mass.copy_(torch.from_numpy(mass))
    s.search_fluid()
    st = s.state()
    g = O.grid(p.cell_size, p.cell_length, hash_rcp=s.device_rcp(p.cell_length))
    A = O.SceneArrays(st["pos"], mass, st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius)
    vb = np.zeros((s.boundary.n, 3))
    if bodies:
        moving = _np(s.body_local())[:, 3] > 0
        vb[moving] = _np(s.boundary.vel)[moving]
        assert np.abs(vb).max() > 0.1
    return s, ref64.Pairs(A), vb, mass


def _set_vel(s, v):
    import torch
    s.fluid.vel.copy_(torch.from_numpy(np.ascontiguousarray(v, F)))
    s.refresh()
    s.search_fluid()


# ---- 1. the two sweeps per element on every path --------------------------------------------------------------------------
@pytest.mark.parametrize("path", sorted(SD.PATHS))
@pytest.mark.parametrize("scene", SCENES)
def test_setup_and_matvec_per_element(pkg, built, scene, path):
    _gpu()
    import torch
    case, bodies = _case(pkg, scene)
    s, P, vb, _ = _system(pkg, case, bodies, SD.PATHS[path])
    p = case.sc.params
    n = s.fluid.n
    try:
        rng = np.random.default_rng(7)
        vel = (0.5 * np.sin(7.0 * s.state()["pos"]) + 0.05 * rng.standard_normal((n, 3))).astype(F)
        _set_vel(s, vel)
        d6 = torch.zeros((n, 6), dtype=torch.float32, device=s.device)
        b = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
        s.visc_implicit_setup(d6, b, NU, NU_B)
        D, mD, bref, mb = IV.setup(P, vel, vb, NU, NU_B, p.dt, p.rho0, p.rho_boundary)
        dg, bg = _np(d6), _np(b)
        tag = f"{scene}/{path}"
        ref64.assert_per_element(dg, ref64.R64(IV.packed(D), IV.packed(mD)), ref64.TAU, tag + " D", ref64.f32_spacing(dg))
        ref64.assert_per_element(bg, ref64.R64(bref, mb), ref64.TAU, tag + " b", ref64.f32_spacing(bg))
        if scene == "body" or (scene == "walls" and n > 1):
            assert np.abs(IV.packed(D) - np.tile([1, 1, 1, 0, 0, 0], (n, 1))).max() > 1e-3, "D is the identity"
        if scene == "body":
            assert np.abs(bref - vel).max() > 1e-4, "the moving body does not enter b"
        # matvec with the GPU's D and a random direction; the records' velocities are left as the API array holds them
        pdir = rng.standard_normal((n, 3)).astype(F)
        ap = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
        s.visc_implicit_matvec(d6, torch.from_numpy(pdir).to(s.device), ap, NU)
        apr, mapr = IV.matvec(P, IV.unpacked(dg), pdir, NU, p.dt, p.rho0)
        apg = _np(ap)
        ref64.assert_per_element(apg, ref64.R64(apr, mapr), ref64.TAU, tag + " A p", ref64.f32_spacing(apg))
        if n > 1:
            assert np.abs(apr - pdir).max() > 1e-4, "A is the identity"
        s.visc_implicit_setup(d6, b, NU, NU_B)           # (b reads the particle's own record velocity: v* again)
        assert np.array_equal(bits(_np(b)), bits(bg)), "records' velocities not restored after the matvec"
    finally:
        s.close()


# ---- 2. the solve against the float64 solution ----------------------------------------------------------------------------
def _solve(pkg, scene, nu, nu_b, tol, max_iter, vel_fn, path="list"):
    case, bodies = _case(pkg, scene)
    s, P, vb, mass = _system(pkg, case, bodies, SD.PATHS[path])
    p = case.sc.params
    pos = s.state()["pos"]
    v0 = vel_fn(pos).astype(F)
    _set_vel(s, v0)
    s.implicit_viscosity(nu, nu_b, tol, max_iter)
    out = s.state()["vel"]
    n = s.fluid.n
    ws = _np(s.visc_work)[WORK_D:WORK_D + 12 * n]            # D[6n] | Dinv[6n] of the workspace (sphk_sweeps.cu)
    s.visc_work = None                                         # the stats are the context's: the workspace may be gone
    it, res = s.implicit_viscosity_stats()
    s.close()
    A, D = IV.assemble(P, nu, nu_b, p.dt, p.rho0, p.rho_boundary)
    _, _, b, _ = IV.setup(P, v0, vb, nu, nu_b, p.dt, p.rho0, p.rho_boundary)
    return dict(v0=v0, out=out, it=it, res=res, A=A, D=D, b=b, mass=mass, pos=pos.astype(np.float64), P=P,
                D6=ws[:6 * n].reshape(n, 6), Dinv6=ws[6 * n:].reshape(n, 6))


@pytest.mark.parametrize("scene", ["body", "mini_last"])
def test_solve_against_the_exact_solution(pkg, built, scene):
    _gpu()
    tol = 1e-4
    def vel_fn(x):
        return 0.5 * np.sin(9.0 * x) + np.random.default_rng(3).standard_normal(x.shape) * 0.1
    r = _solve(pkg, scene, 0.1, 0.1, tol, 200, vel_fn)
    A, b, m, x = r["A"], r["b"], r["mass"], r["out"].astype(np.float64)
    resid = IV.m_norm(b - (A @ x.ravel()).reshape(-1, 3), m) / IV.m_norm(b, m)
    assert resid <= tol * 1.05, resid
    assert r["res"] <= tol and r["res"] > 0
    _, it64, _ = IV.pcg(A, r["D"], b, r["v0"], m, tol, 200)
    assert it64 >= 2 and abs(r["it"] - it64) <= 1, (r["it"], it64)
    exact = IV.solve(A, b)
    lam_min = IV.spectrum(A, m, "SA")
    assert lam_min >= 1.0 - 1e-9
    err = IV.m_norm(x - exact, m)
    assert err <= resid * IV.m_norm(b, m) / lam_min * (1 + 1e-6), (err, resid)
    assert not np.array_equal(bits(r["out"]), bits(r["v0"]))
    # the reported residual is the M-norm one, and the loop ends at the FIRST iteration that meets the test: stopped one
    # iteration earlier by max_iter, the same solve is still above tol
    assert abs(r["res"] - resid) <= 0.05 * resid, (r["res"], resid)
    early = _solve(pkg, scene, 0.1, 0.1, tol, r["it"] - 1, vel_fn)
    assert early["it"] == r["it"] - 1 and early["res"] > tol, (early["it"], early["res"])


@pytest.mark.parametrize("scene,nu,nu_b,variant", [("wide", 0.1, 0.1, "euclidean"), ("oblique", 0.02, 1.0, "diagonal")])
def test_solve_tells_the_preconditioner_and_the_inner_product_apart(pkg, built, scene, nu, nu_b, variant):
    """Scenes where the float64 PCG with Euclidean dot products (masses over a factor 49) or with the diagonal of D_i as the
    preconditioner (an oblique plate with a large nu_b: D_i anisotropic off the axes) needs at least 2 more iterations than
    the engine's (M inner product, block Jacobi): the GPU count is the engine variant's +-1, and the workspace's D_i^-1 is the
    inverse of its D_i per element"""
    _gpu()
    tol = 1e-4

    def vel_fn(x):
        return 0.5 * np.sin(9.0 * x) + np.random.default_rng(3).standard_normal(x.shape) * 0.1
    r = _solve(pkg, scene, nu, nu_b, tol, 200, vel_fn)
    A, b, m = r["A"], r["b"], r["mass"]
    _, it_m, _ = IV.pcg(A, r["D"], b, r["v0"], m, tol, 500)
    _, it_v, _ = IV.pcg(A, r["D"], b, r["v0"], m, tol, 500, precond="diag" if variant == "diagonal" else "block",
                        weighted=variant != "euclidean")
    assert it_v >= it_m + 2, (it_m, it_v)
    assert abs(r["it"] - it_m) <= 1, (r["it"], it_m, it_v)
    x = r["out"].astype(np.float64)
    resid = IV.m_norm(b - (A @ x.ravel()).reshape(-1, 3), m) / IV.m_norm(b, m)
    assert resid <= tol * 1.05 and abs(r["res"] - resid) <= 0.05 * resid, (r["res"], resid)
    inv = IV.packed(np.linalg.inv(IV.unpacked(r["D6"])))
    scale = np.abs(inv).max(1, keepdims=True)
    assert np.all(np.abs(r["Dinv6"] - inv) <= 1e-5 * scale), np.abs(r["Dinv6"] - inv).max()
    if variant == "diagonal":
        assert (np.abs(inv[:, 3:]) > 0.05 * inv[:, :3].min(1, keepdims=True)).any(), "D^-1 is nearly diagonal everywhere"


# ---- 3. momentum and energy -----------------------------------------------------------------------------------------------
def _clear_block(pkg):
    """a jittered block in the middle of the mini box, more than R from every wall"""
    sc = pkg.scene.make_scene("mini", solver="dfsph", max_iter=4, den_thr=-1.0, div_thr=-1.0)
    g = np.arange(9) * 0.02 + 0.16
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    pos = pos + np.random.default_rng(2).uniform(-0.003, 0.003, pos.shape)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(pos.astype(F)))


def test_momentum_and_energy_clear_of_the_walls(pkg, built, monkeypatch):
    _gpu()
    sc = _clear_block(pkg)
    monkeypatch.setattr(SD, "make_case", lambda pkg_, name: SD.Case(name, sc, mass="random", lattice_like=False))
    r = _solve(pkg, "clear", 0.1, 0.0, 1e-6, 200, lambda x: np.random.default_rng(9).standard_normal(x.shape))
    assert r["P"].iB.size == 0
    m, x, v0, pos = r["mass"].astype(np.float64), r["out"].astype(np.float64), r["v0"].astype(np.float64), r["pos"]
    rr = IV.m_norm(r["b"] - (r["A"] @ x.ravel()).reshape(-1, 3), m)
    dp = np.abs((m[:, None] * (x - v0)).sum(0)).max()
    dL = np.abs((m[:, None] * (np.cross(pos, x) - np.cross(pos, v0))).sum(0)).max()
    # the exact solution conserves both: the change is that of the error, |e|_M <= |r|_M (eigenvalues >= 1)
    assert dp <= np.sqrt(m.sum()) * rr * 1.01 + 1e-9, (dp, rr)
    assert dL <= np.sqrt((m * (pos ** 2).sum(1)).sum()) * rr * 1.01 + 1e-9, (dL, rr)
    assert np.abs(x - v0).max() > 1e-2
    assert (m[:, None] * x * x).sum() <= (m[:, None] * v0 * v0).sum()
    # a rigid rotation: r0 is rounding only -> no iteration, the velocities come out unchanged
    c = pos.mean(0)
    r = _solve(pkg, "clear", 0.1, 0.0, 1e-4, 200, lambda q: np.cross([0.3, 2.0, -0.5], q - c) + [0.1, 0.0, 0.2])
    assert r["it"] == 0
    assert np.array_equal(bits(r["out"]), bits(r["v0"]))


# ---- 4. a fluid at rest ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["walls", "config0", "n1"])
def test_fluid_at_rest_is_unchanged(pkg, built, scene):
    _gpu()
    r = _solve(pkg, scene, 0.2, 0.2, 1e-4, 50, lambda x: np.zeros_like(x))
    assert r["it"] == 0 and r["res"] == 0.0
    assert np.all(r["out"] == 0) and np.array_equal(bits(r["out"]), bits(r["v0"]))


def test_fluid_at_rest_after_the_constructors_step_0(pkg, built):
    """a system that has taken step 0 (no gravity): with its velocities at rest the solve takes 0 iterations and keeps the bits"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene("mini", solver="dfsph", max_iter=4, den_thr=-1.0, div_thr=-1.0)
    sc = dataclasses.replace(sc, params=dataclasses.replace(sc.params, gravity=(0.0, 0.0, 0.0)))
    s = engine.SphkSystem(sc)
    s.fluid.vel.zero_()
    s.refresh()
    s.implicit_viscosity(0.2, 0.2)
    v = s.state()["vel"]
    assert s.implicit_viscosity_stats() == (0, 0.0)
    assert np.all(v == 0) and not np.signbit(v).any()
    s.close()


def test_stats_before_any_solve_and_after_the_constructor(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    app = capi.SphApp(pkg.scene.benchmark_scene("mini", "dfsph"))
    assert app.viscosity_stats() == (0, 0.0)
    app.set_implicit_viscosity(0.05, 0.05)
    app.step()
    it, res = app.viscosity_stats()
    assert it >= 1 and 0 < res <= 1e-4
    app.close()


# ---- 5. off means off, the step graph -------------------------------------------------------------------------------------
def _app(pkg, solver, scene="mini"):
    from cpp_fluid_particles_b200 import capi
    return capi.SphApp(pkg.scene.benchmark_scene(scene, solver))


def _same(a, b, what, fields=("pos", "vel", "density")):
    for f in fields:
        assert np.array_equal(bits(a[f]), bits(b[f])), f"{what}: {f} differs"


@pytest.mark.parametrize("solver", SOLVERS)
def test_off_means_off(pkg, built, solver):
    """nu = 0 (never set, set, or toggled back) is today's step: same bits, same launches per step"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    a, b, c = _app(pkg, solver), _app(pkg, solver), _app(pkg, solver)
    b.set_implicit_viscosity(0.0)
    c.set_implicit_viscosity(NU, NU_B); c.set_implicit_viscosity(0.0, NU_B)
    sc = pkg.scene.benchmark_scene("mini", solver)
    e0, e1 = engine.SphkSystem(sc), engine.SphkSystem(sc)
    e1.implicit_nu, e1.implicit_nu_boundary = 0.0, NU_B
    for k in range(4):
        for x in (a, b, c):
            x.step()
        l0, l1 = e0.launch_count(), e1.launch_count()
        e0.step(); e1.step()
        assert e0.launch_count() - l0 == e1.launch_count() - l1
        ra = a.download()
        _same(ra, b.download(), f"{solver} step {k} nu=0 set")
        _same(ra, c.download(), f"{solver} step {k} nu toggled back to 0")
        _same(ra, e0.state(), f"{solver} step {k} python engine", ("pos", "density"))
        _same(e0.state(), e1.state(), f"{solver} step {k} python engine nu=0")
    e1.implicit_nu = NU
    l0, l1 = e0.launch_count(), e1.launch_count()
    e0.step(); e1.step()
    assert e1.launch_count() - l1 > e0.launch_count() - l0, "nu > 0 runs the solve"
    for x in (a, b, c, e0, e1):
        x.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_step_graph_with_implicit_viscosity(pkg, built, solver):
    """graph on and off give the same bits with the solve on, and changing nu between steps drops the captured graph"""
    _gpu()
    g, p = _app(pkg, solver), _app(pkg, solver)
    p.set_option(3, 0)
    schedule = [NU] * 4 + [0.0] * 2 + [0.2] * 3 + [NU] * 2
    for k, nu in enumerate(schedule):
        g.set_implicit_viscosity(nu, NU_B); p.set_implicit_viscosity(nu, NU_B)
        g.step(); p.step()
        _same(g.download(), p.download(), f"{solver} step {k} (nu {nu}): graph vs plain launches")
        assert g.viscosity_stats() == p.viscosity_stats()
    assert g.step_graph_active() and not p.step_graph_active()
    g.close(); p.close()


# ---- 6. the layers agree --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_layers_agree(pkg, built, tmp_path, solver):
    """nu = nu_b > 0: facade (class layer), python engine and sph_headless --implicit-viscosity give the same bits over 3
    frames; the solve changes the result"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", solver)
    app, off = _app(pkg, solver), _app(pkg, solver)
    app.set_implicit_viscosity(NU, NU)
    s = engine.SphkSystem(sc)
    s.implicit_nu = s.implicit_nu_boundary = NU
    for k in range(3):
        app.step(); s.step(); off.step()
        a = app.download()
        _same(a, s.state(), f"{solver} frame {k}: facade vs python engine")
        assert app.viscosity_stats() == s.implicit_viscosity_stats()
    assert not np.array_equal(bits(a["vel"]), bits(off.download()["vel"])), "the solve must change the velocities"
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    prefix = str(tmp_path / "dump")
    cmd = [CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--frames", "3", "--box", str(box), "--block", str(nx), str(ny),
           str(nz), "--origin", *[repr(float(o)) for o in origin], "--dump", prefix, "--quiet", "--implicit-viscosity", repr(NU)]
    if solver != "wcsph":
        cmd += ["--iters", "4"]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    pos = np.fromfile(prefix + ".pos.f32", np.float32).reshape(-1, 3)
    den = np.fromfile(prefix + ".density.f32", np.float32)
    assert np.array_equal(bits(pos), bits(a["pos"])) and np.array_equal(bits(den), bits(a["density"])), "sph_headless"
    app.close(); off.close(); s.close()


# ---- 7. validation --------------------------------------------------------------------------------------------------------
def test_entries_validate_arguments(pkg, built):
    _gpu()
    import ctypes as C
    import torch
    from cpp_fluid_particles_b200 import engine
    from cpp_fluid_particles_b200.engine import _ptr
    s = engine.SphkSystem(pkg.scene.make_scene("mini", "dfsph"), step0=False)
    L, ctx, sc = s.L, s.ctx, s._s()
    w = s._visc_work()
    INVALID, STATE = -1, -4
    f, i = C.c_float, C.c_int

    def solve(work=w, nu=NU, nub=NU_B, dt=0.004, rho0=1.0, rhob=1.4, tol=1e-4, it=10):
        return L.sphk_implicit_viscosity(ctx, sc, work, f(nu), f(nub), f(dt), f(rho0), f(rhob), f(tol), i(it))

    nan = float("nan")
    assert solve(work=None) == INVALID
    assert solve(work=_ptr(s.fluid.vel)) == INVALID
    for kw in ({"nu": -0.1}, {"nu": nan}, {"nub": -0.1}, {"nub": nan}, {"rho0": 0.0}, {"rho0": -1.0}, {"tol": 0.0}, {"tol": -1e-4},
               {"tol": nan}, {"it": 0}, {"it": -3}, {"it": 1001}):
        assert solve(**kw) == INVALID, kw
    assert solve() == 0 and solve(it=1000) == 0
    n = s.fluid.n
    d6 = torch.zeros((n, 6), dtype=torch.float32, device=s.device)
    b = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
    ap = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
    setup = lambda dd, bb, nu=NU: L.sphk_visc_implicit_setup(ctx, sc, dd, bb, f(nu), f(NU_B), f(0.004), f(1.0), f(1.4))  # noqa: E731
    matvec = lambda dd, pp, aa, nu=NU: L.sphk_visc_implicit_matvec(ctx, sc, dd, pp, aa, f(nu), f(0.004), f(1.0))  # noqa: E731
    assert setup(None, _ptr(b)) == INVALID and setup(_ptr(d6), None) == INVALID and setup(_ptr(d6), _ptr(d6)) == INVALID
    assert setup(_ptr(d6), _ptr(b), nu=-1.0) == INVALID
    assert matvec(_ptr(d6), None, _ptr(ap)) == INVALID and matvec(_ptr(d6), _ptr(b), _ptr(b)) == INVALID
    assert matvec(_ptr(d6), _ptr(b), _ptr(s.fluid.vel)) == INVALID
    assert setup(_ptr(d6), _ptr(b)) == 0 and matvec(_ptr(d6), _ptr(b), _ptr(ap)) == 0
    # an active range (slab ranks)
    L.sphk_set_active_range(ctx, i(0), i(n // 2))
    assert solve() == STATE and setup(_ptr(d6), _ptr(b)) == STATE and matvec(_ptr(d6), _ptr(b), _ptr(ap)) == STATE
    L.sphk_set_active_range(ctx, i(0), i(-1))
    assert solve() == 0
    s.close()
    # dynamic bodies: nu_b > 0 is refused (the viscous wall force is not part of their reaction); nu_b = 0 runs
    sc2 = pkg.scene.make_scene("mini", "dfsph")
    body = dict(_plate(sc2.fluid.mean(0), v=(0, 0, 0), w=(0, 0, 0)), mass=0.01, inertia=[1e-4, 1e-4, 1e-4])
    s = engine.SphkSystem(sc2, step0=False, bodies=[body])
    assert s.bodies_dynamic
    w = s._visc_work()
    assert s.L.sphk_implicit_viscosity(s.ctx, s._s(), w, f(NU), f(NU_B), f(0.004), f(1.0), f(1.4), f(1e-4), i(10)) == STATE
    assert s.L.sphk_implicit_viscosity(s.ctx, s._s(), w, f(NU), f(0.0), f(0.004), f(1.0), f(1.4), f(1e-4), i(10)) == 0
    s.close()


def test_facade_validates_arguments(pkg, built):
    _gpu()
    app = _app(pkg, "dfsph")
    for args in ((-0.1, 0.0), (float("nan"), 0.0), (0.1, -1.0), (0.1, 0.0, 0.0), (0.1, 0.0, 1e-4, 0), (0.1, 0.0, 1e-4, 1001)):
        with pytest.raises(RuntimeError):
            app.set_implicit_viscosity(*args)
    app.close()


def test_dynamic_bodies_refuse_a_boundary_viscosity(pkg, built):
    """with a dynamic body the facade (and the class layer under it) refuses nu_b > 0 and keeps the setting: every step then
    still runs the solve it was given"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    body = dict(_plate(sc.fluid.mean(0), v=(0, 0, 0), w=(0, 0, 0)), mass=0.01, inertia=[1e-4, 1e-4, 1e-4])
    app = capi.SphApp(sc, bodies=[body])
    app.set_implicit_viscosity(0.05, 0.0)
    with pytest.raises(RuntimeError):
        app.set_implicit_viscosity(0.05, 0.05)
    app.step()
    it, res = app.viscosity_stats()
    assert it >= 1 and 0 < res <= 1e-4
    app.close()


# ---- 8. physics -----------------------------------------------------------------------------------------------------------
def _dam(pkg, nu, steps):
    """mini DFSPH dam break with nu = nu_b from the first step on; (positions, velocities, max KE over the run)"""
    app = _app(pkg, "dfsph")
    app.set_implicit_viscosity(nu, nu)
    m = app.download()["mass"].astype(np.float64)
    ke = []
    for _ in range(steps):
        app.step()
        v = app.download()["vel"].astype(np.float64)
        ke.append(0.5 * (m * (v ** 2).sum(1)).sum())
    st = app.download()
    app.close()
    return st, np.array(ke)


def test_dam_break_far_above_the_explicit_limit_stays_finite(pkg, built):
    """nu = 12.5 nu_crit (the explicit step of the same operator is unstable above nu_crit): 200 steps, finite, and the kinetic
    energy stays below the potential energy the block can release"""
    _gpu()
    nu = 12.5 * NU_CRIT_MINI
    st, ke = _dam(pkg, nu, 200)
    assert np.isfinite(st["pos"]).all() and np.isfinite(st["vel"]).all() and np.isfinite(ke).all()
    m = st["mass"].astype(np.float64)
    pe = (m * 9.8 * 0.32).sum()                                # no particle can fall further than the block's top, 0.315
    assert ke.max() <= pe, (ke.max(), pe)
    assert np.abs(st["vel"]).max() < 5.0


def test_dam_break_front_advances_less_for_larger_viscosity(pkg, built):
    _gpu()
    spread = []
    for nu in (0.001, 0.03, 0.3):
        st, _ = _dam(pkg, nu, 30)
        x = st["pos"][:, [0, 2]].astype(np.float64)
        spread.append(float(np.abs(x - x.mean(0)).mean()))
    print(f"\nmean horizontal distance from the centre after 30 steps, nu = 0.001 / 0.03 / 0.3: {spread}")
    assert spread[0] > spread[1] > spread[2], spread


def test_paddle_drags_the_fluid_with_a_no_slip_boundary(pkg, built):
    """a plate rotating about y through the mini block: with nu_b > 0 the fluid near it picks up angular momentum with the sign
    of Omega faster than with nu_b = 0 (the same nu)"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    c = sc.fluid.mean(0)
    body = _plate(c, v=(0.0, 0.0, 0.0), w=(0.0, 10.0, 0.0))
    keep = np.abs(sc.fluid[:, 2] - c[2]) > 0.02
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(sc.fluid[keep]))
    out = []
    for nub in (0.0, 0.05):
        app = capi.SphApp(sc, bodies=[body])
        app.set_implicit_viscosity(0.05, nub)
        for _ in range(8):
            app.step()
        st = app.download()
        app.close()
        x, v, m = st["pos"].astype(np.float64) - c, st["vel"].astype(np.float64), st["mass"].astype(np.float64)
        near = np.sqrt(x[:, 0] ** 2 + x[:, 2] ** 2) < 0.08
        out.append(float((m * (x[:, 2] * v[:, 0] - x[:, 0] * v[:, 2]))[near].sum()))
    print(f"\nL_y near the paddle after 8 steps: nu_b = 0: {out[0]:.4g}, nu_b = 0.05: {out[1]:.4g}")
    assert out[1] > 0 and out[1] > out[0], out


# ---- 9. sph_headless --implicit-viscosity with blocking launches (memcheck with SPHK_SANITIZER=1) ------------------------------
@pytest.mark.parametrize("solver", ["sph", "dfsph", "pbd"])
@pytest.mark.parametrize("stir", [False, True])
def test_headless_runs_cleanly(built, tmp_path, solver, stir):
    _gpu()
    cmd = [CLI, "--solver", solver, "--frames", "3", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055",
           "0.135", "--quiet", "--implicit-viscosity", "0.05"] + (["--iters", "2"] if solver != "sph" else []) + \
          (["--stir", "6"] if stir else [])
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
