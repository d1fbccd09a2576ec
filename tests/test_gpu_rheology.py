"""Non-Newtonian viscosity on the GPU: the shear sweep per element on every execution path against the float64 reference
(tests/rheology_ref.py), the models on given shear rates, the setup and matvec sweeps with a per-particle viscosity, the solve
against the float64 PCG, a Newtonian Cross fluid against the constant-nu solve, off means off, the step graph, the four layers,
argument validation, the physics of a Bingham and a Cross dam break, and sph_headless --rheology."""
import os
import subprocess

import numpy as np
import pytest

import implicit_visc_ref as IV
import ref64
import rheology_ref as RR
import sweep_driver as SD
import test_gpu_implicit_viscosity as TIV
from util import bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
SCENES = TIV.SCENES
CROSS = dict(model="cross", nu0=0.3, nu_inf=0.01, lam=0.5, m=1.0, nu_max=0.3)
BINGHAM = dict(model="hb", k=0.02, n=1.0, tau_y=0.3, m_reg=100.0, nu_max=0.5)
_gpu, _np, _case, _system, _set_vel, _same = TIV._gpu, TIV._np, TIV._case, TIV._system, TIV._set_vel, TIV._same


def _params(spec):
    from cpp_fluid_particles_b200 import capi
    r = capi.rheology(spec)
    return r.model, [float(x) for x in r.params], float(r.nu_min), float(r.nu_max)


def _model64(spec, g):
    model, params, lo, hi = _params(spec)
    return RR.model_nu(model, params, lo, hi, g)


def _ulps(x, ref):
    """|x - ref| in units of the float32 spacing at ref"""
    x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
    sp = np.spacing(np.abs(ref.astype(np.float32))).astype(np.float64)
    sp = np.where(sp > 0, sp, np.spacing(np.float32(0)))
    return np.abs(x - ref) / sp


def _vel(pos, seed=7):
    rng = np.random.default_rng(seed)
    return (0.5 * np.sin(7.0 * pos) + 0.05 * rng.standard_normal(pos.shape)).astype(F)


# ---- 1. the shear sweep per element on every path ---------------------------------------------------------------------------
def _shear(s, spec, beta):
    import torch
    n = s.fluid.n
    z = lambda *shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device=s.device)  # noqa: E731
    gam, nu, grad, flag = z(n), z(n), z(n, 9), z(n, dt=torch.int32)
    s.shear_rate(gam, nu, spec, grad, flag, beta)
    return _np(gam), _np(nu), _np(grad).reshape(n, 3, 3), _np(flag)


@pytest.mark.parametrize("path", sorted(SD.PATHS))
@pytest.mark.parametrize("scene", SCENES)
def test_shear_rate_per_element(pkg, built, scene, path):
    """gamma_dot, grad v (9 floats) and the branch flag against the float64 sweep, 2e-6 mag + the float32 floor; where det M_i is
    within rounding of the switch either branch is accepted.  nu = the float64 model of the GPU's own gamma_dot within 2 ulp, and
    the statistics are those of the arrays."""
    _gpu()
    case, bodies = _case(pkg, scene)
    s, P, vb, _ = _system(pkg, case, bodies, SD.PATHS[path])
    p = case.sc.params
    try:
        vel = _vel(s.state()["pos"])
        _set_vel(s, vel)
        beta = 1.0
        gam, nu, grad, flag = _shear(s, BINGHAM, beta)
        ref = RR.shear(P, vel, vb, beta, p.rho0, p.rho_boundary)
        tag = f"{scene}/{path}"
        near = ref["near"]
        assert np.array_equal(flag[~near], ref["flag"][~near]), f"{tag}: branch flags differ"
        gm = np.maximum(ref["grad_mag"], ref["grad_alt_mag"])
        ref64.assert_per_element(grad, ref64.R64(ref["grad"], gm, ref["grad_alt"]), ref64.TAU, tag + " grad v",
                                 ref64.f32_spacing(grad))
        ref64.assert_per_element(gam, ref64.R64(ref["gamma"], np.maximum(ref["gamma_mag"], ref["gamma_alt_mag"]), ref["gamma_alt"]),
                                 ref64.TAU, tag + " gamma_dot", ref64.f32_spacing(gam))
        want, at = _model64(BINGHAM, gam)
        assert _ulps(nu, want).max() <= 2.0, f"{tag}: nu"
        st = s.non_newtonian_stats()
        assert st["gamma_max"] == float(gam.max()) and st["nu_min"] == float(nu.min()) and st["nu_max"] == float(nu.max())
        assert st["at_nu_max"] == int(at.sum())
        if case.lattice_like:
            assert (flag == 0).mean() > 0.9 and gam.max() > 1.0
        if scene == "n1":
            assert flag[0] == 1 and gam[0] == 0.0
        if scene in ("walls", "body") and s.fluid.n > 1:
            # the boundary pairs enter the gradient: beta = 0 gives another gradient next to the walls
            g0, _, _, _ = _shear(s, BINGHAM, 0.0)
            r0 = RR.shear(P, vel, vb, 0.0, p.rho0, p.rho_boundary)
            ref64.assert_per_element(g0, ref64.R64(r0["gamma"], np.maximum(r0["gamma_mag"], r0["gamma_alt_mag"]), r0["gamma_alt"]),
                                     ref64.TAU, tag + " gamma_dot (beta = 0)", ref64.f32_spacing(g0))
            assert np.abs(r0["gamma"] - ref["gamma"]).max() > 1e-3
    finally:
        s.close()


def test_linear_field_gives_its_gradient_on_the_gpu(pkg, built):
    """the closed form through the kernel: v = A x + b on the fluid and the wall records of the mini scene"""
    _gpu()
    case, _ = _case(pkg, "walls")
    s, P, vb, _ = _system(pkg, case, None)
    try:
        A = np.array([[0.3, -1.2, 0.5], [0.8, 0.1, -0.4], [-0.6, 0.9, 0.2]])
        pos = s.state()["pos"].astype(np.float64)
        _set_vel(s, pos @ A.T + [0.1, 0.2, -0.3])
        _, _, grad, flag = _shear(s, BINGHAM, 0.0)
        ok = (flag == 0) & (np.bincount(P.iF, minlength=P.n) >= 8)
        assert ok.mean() > 0.9
        assert np.abs(grad[ok] - A[None]).max() <= 2e-4 * np.abs(A).max(), np.abs(grad[ok] - A[None]).max()
    finally:
        s.close()


# ---- 2. the models on given shear rates -------------------------------------------------------------------------------------
MODELS = [CROSS, dict(CROSS, nu0=0.05, nu_inf=0.05), dict(model="cross", nu0=0.01, nu_inf=0.3, lam=2.0, m=2.0, nu_max=1e30),
          BINGHAM, dict(model="hb", k=0.1, n=0.4, tau_y=0.0, nu_max=1e30), dict(model="hb", k=0.1, n=1.6, tau_y=0.0, nu_max=1e30),
          dict(model="hb", k=0.0, n=1.0, tau_y=2.0, m_reg=50.0, nu_max=1e30, nu_min=1e-3)]


@pytest.mark.parametrize("k", range(len(MODELS)))
def test_rheology_eval_within_two_ulp(pkg, built, k):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    spec = MODELS[k]
    g = np.concatenate([[0.0, 1e-45, 1e-40, 1e-38, 1e-30, 1e30, 3e38], 10.0 ** np.random.default_rng(k).uniform(-8, 8, 4000)])
    g = g.astype(F)
    s = engine.SphkSystem(pkg.scene.make_scene("mini", "dfsph"), step0=False)
    try:
        out = torch.zeros(g.size, dtype=torch.float32, device=s.device)
        s.rheology_eval(spec, torch.from_numpy(g).to(s.device), out)
        x = _np(out)
        want, _ = _model64(spec, g.astype(np.float64))
        u = _ulps(x, want)
        assert u.max() <= 2.0, (u.max(), g[u.argmax()], x[u.argmax()], want[u.argmax()])
        if spec["model"] == "hb" and spec["tau_y"] > 0:
            assert x[0] == F(min(spec["tau_y"] * spec.get("m_reg", 1000.0) + spec["k"], spec["nu_max"]))
    finally:
        s.close()


# ---- 3. setup and matvec with a per-particle nu -----------------------------------------------------------------------------
def _nu_field(n, seed=11):
    return (0.001 * np.exp(np.random.default_rng(seed).uniform(0.0, np.log(1000.0), n))).astype(F)


def _field_sweeps(s, P, vb, vel, nu, beta, p):
    import torch
    n = s.fluid.n
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(s.device)  # noqa: E731
    d6 = torch.zeros((n, 6), dtype=torch.float32, device=s.device)
    b = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
    s.visc_field_setup(d6, b, t(nu), beta)
    pdir = np.random.default_rng(3).standard_normal((n, 3)).astype(F)
    ap = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
    s.visc_field_matvec(d6, t(pdir), ap, t(nu))
    return _np(d6), _np(b), pdir, _np(ap)


@pytest.mark.parametrize("path", sorted(SD.PATHS))
@pytest.mark.parametrize("scene", SCENES)
def test_field_setup_and_matvec_per_element(pkg, built, scene, path):
    """nu log-uniform over a factor of 1000, beta = 1 (0 on the list path): D_i, b_i and (A p)_i against float64"""
    _gpu()
    case, bodies = _case(pkg, scene)
    s, P, vb, _ = _system(pkg, case, bodies, SD.PATHS[path])
    p = case.sc.params
    try:
        n = s.fluid.n
        vel = _vel(s.state()["pos"])
        _set_vel(s, vel)
        nu = _nu_field(n)
        for beta in ((1.0, 0.0) if path == "list" else (1.0,)):
            dg, bg, pdir, apg = _field_sweeps(s, P, vb, vel, nu, beta, p)
            D, mD, bref, mb = RR.setup(P, vel, vb, nu, beta, p.dt, p.rho0, p.rho_boundary)
            tag = f"{scene}/{path}/beta={beta}"
            ref64.assert_per_element(dg, ref64.R64(IV.packed(D), IV.packed(mD)), ref64.TAU, tag + " D", ref64.f32_spacing(dg))
            ref64.assert_per_element(bg, ref64.R64(bref, mb), ref64.TAU, tag + " b", ref64.f32_spacing(bg))
            apr, mapr = RR.matvec(P, IV.unpacked(dg), pdir, nu, p.dt, p.rho0)
            ref64.assert_per_element(apg, ref64.R64(apr, mapr), ref64.TAU, tag + " A p", ref64.f32_spacing(apg))
            if n > 1:
                assert np.abs(apr - pdir).max() > 1e-4, "A is the identity"
        assert np.array_equal(bits(s.state()["vel"]), bits(vel)), "the matvec did not restore the records' velocities"
    finally:
        s.close()


@pytest.mark.parametrize("scene", ["config0_mass", "mini_last", "body"])
def test_operator_is_self_adjoint_only_with_the_mean(pkg, built, scene):
    """<u, A w>_M = <A u, w>_M in float64 with nu_ij = (nu_i + nu_j) / 2; nu_j instead of the mean breaks it"""
    _gpu()
    case, bodies = _case(pkg, scene)
    s, P, vb, mass = _system(pkg, case, bodies)
    p = case.sc.params
    s.close()
    nu = _nu_field(P.n)
    rng = np.random.default_rng(4)
    u, w = rng.standard_normal((2, 3 * P.n))
    rel = []
    for mean in (True, False):
        A, _ = RR.assemble(P, nu, 1.0, p.dt, p.rho0, p.rho_boundary, mean=mean)
        lhs, rhs = RR.m_dot(u, A @ w, mass), RR.m_dot(A @ u, w, mass)
        rel.append(abs(lhs - rhs) / (abs(lhs) + abs(rhs)))
    assert rel[0] <= 1e-12 and rel[1] >= 1e-6, rel


# ---- 4. the solve -----------------------------------------------------------------------------------------------------------
def _solve(pkg, scene, spec, vel_fn, path="list"):
    case, bodies = _case(pkg, scene)
    s, P, vb, mass = _system(pkg, case, bodies, SD.PATHS[path])
    p = case.sc.params
    pos = s.state()["pos"]
    v0 = vel_fn(pos).astype(F)
    _set_vel(s, v0)
    s.non_newtonian_viscosity(spec)
    out = s.state()["vel"]
    nu = _np(s.nu_field)[:s.fluid.n]
    s.rheo_work = None                                           # the stats are the context's: the workspace may be gone
    st = s.non_newtonian_stats()
    s.close()
    beta = spec.get("beta", 0.0)
    A, D = RR.assemble(P, nu, beta, p.dt, p.rho0, p.rho_boundary)
    _, _, b, _ = RR.setup(P, v0, vb, nu, beta, p.dt, p.rho0, p.rho_boundary)
    return dict(v0=v0, out=out, nu=nu, st=st, A=A, D=D, b=b, mass=mass, pos=pos.astype(np.float64), P=P, vb=vb, p=p)


@pytest.mark.parametrize("scene,spec", [("body", dict(CROSS, beta=1.0, max_iter=200)), ("mini_last", dict(BINGHAM, beta=1.0, max_iter=200)),
                                        ("walls", dict(BINGHAM, beta=0.0, max_iter=200))])
def test_solve_against_the_float64_pcg(pkg, built, scene, spec):
    _gpu()
    tol = spec.get("tol", 1e-4)

    def vel_fn(x):
        return 0.5 * np.sin(9.0 * x) + np.random.default_rng(3).standard_normal(x.shape) * 0.1
    r = _solve(pkg, scene, spec, vel_fn)
    A, b, m, x = r["A"], r["b"], r["mass"], r["out"].astype(np.float64)
    assert r["nu"].max() / max(r["nu"].min(), 1e-30) > 3.0, "the viscosity does not vary"
    resid = IV.m_norm(b - (A @ x.ravel()).reshape(-1, 3), m) / IV.m_norm(b, m)
    assert resid <= tol * 1.05, resid
    _, it64, _ = IV.pcg(A, r["D"], b, r["v0"], m, tol, 200)
    it = r["st"]["iterations"]
    print(f"\n{scene}: {it} iterations (float64 PCG {it64}), nu in [{r['nu'].min():.3g}, {r['nu'].max():.3g}]")
    assert it64 >= 2 and abs(it - it64) <= 1, (it, it64)
    assert 0 < r["st"]["residual"] <= tol


@pytest.mark.parametrize("scene", ["walls", "config0", "n1"])
def test_fluid_at_rest_is_unchanged(pkg, built, scene):
    _gpu()
    r = _solve(pkg, scene, dict(BINGHAM, beta=1.0), lambda x: np.zeros_like(x))
    assert r["st"]["iterations"] == 0 and r["st"]["residual"] == 0.0
    assert np.all(r["out"] == 0) and np.array_equal(bits(r["out"]), bits(r["v0"]))
    assert r["st"]["gamma_max"] == 0.0 and np.all(r["nu"] == F(BINGHAM["nu_max"]))     # at rest a Bingham fluid is unyielded


def test_momentum_clear_of_the_walls(pkg, built, monkeypatch):
    """beta = 0, no boundary neighbour: linear and angular momentum change by no more than the residual allows"""
    _gpu()
    sc = TIV._clear_block(pkg)
    monkeypatch.setattr(SD, "make_case", lambda pkg_, name: SD.Case(name, sc, mass="random", lattice_like=False))
    r = _solve(pkg, "clear", dict(CROSS, tol=1e-6, max_iter=300), lambda x: np.random.default_rng(9).standard_normal(x.shape))
    assert r["P"].iB.size == 0
    m, x, v0, pos = r["mass"].astype(np.float64), r["out"].astype(np.float64), r["v0"].astype(np.float64), r["pos"]
    rr = IV.m_norm(r["b"] - (r["A"] @ x.ravel()).reshape(-1, 3), m)
    dp = np.abs((m[:, None] * (x - v0)).sum(0)).max()
    dL = np.abs((m[:, None] * (np.cross(pos, x) - np.cross(pos, v0))).sum(0)).max()
    assert dp <= np.sqrt(m.sum()) * rr * 1.01 + 1e-9, (dp, rr)
    assert dL <= np.sqrt((m * (pos ** 2).sum(1)).sum()) * rr * 1.01 + 1e-9, (dL, rr)
    assert np.abs(x - v0).max() > 1e-2


# ---- 5. a Newtonian Cross fluid is the constant-nu solve ---------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["body", "walls", "config0_mass"])
def test_newtonian_cross_reproduces_the_constant_nu_solve(pkg, built, scene):
    _gpu()
    nu = 0.05
    spec = dict(model="cross", nu0=nu, nu_inf=nu, lam=1.0, m=1.0, nu_max=nu, beta=1.0, max_iter=100)
    outs = []
    for which in ("rheology", "constant"):
        case, bodies = _case(pkg, scene)
        s, _, _, _ = _system(pkg, case, bodies)
        _set_vel(s, (0.5 * np.sin(9.0 * s.state()["pos"])).astype(F))
        if which == "rheology":
            s.non_newtonian_viscosity(spec)
            it = s.non_newtonian_stats()["iterations"]
        else:
            s.implicit_viscosity(nu, nu, 1e-4, 100)
            it = s.implicit_viscosity_stats()[0]
        outs.append((s.state()["vel"], it))
        s.close()
    (a, ia), (b, ib) = outs
    same = np.array_equal(bits(a), bits(b))
    print(f"\n{scene}: Newtonian Cross vs constant nu: {ia} / {ib} iterations, bit-identical: {same}, "
          f"max |dv| / max |v| = {np.abs(a - b).max() / np.abs(b).max():.3g}")
    assert ia == ib >= 1
    assert np.abs(a.astype(np.float64) - b).max() <= 1e-6 * np.abs(b).max()


# ---- 6. off means off, the step graph ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_off_means_off(pkg, built, solver):
    """never set, and set then cleared, give the same bits and the same launches per step"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    a, c = TIV._app(pkg, solver), TIV._app(pkg, solver)
    c.set_rheology(BINGHAM); c.set_rheology(None)
    sc = pkg.scene.benchmark_scene("mini", solver)
    e0, e1 = engine.SphkSystem(sc), engine.SphkSystem(sc)
    e1.rheology = BINGHAM
    e1.rheology = None
    for k in range(4):
        a.step(); c.step()
        l0, l1 = e0.launch_count(), e1.launch_count()
        e0.step(); e1.step()
        assert e0.launch_count() - l0 == e1.launch_count() - l1
        _same(a.download(), c.download(), f"{solver} step {k} rheology set and cleared")
        _same(e0.state(), e1.state(), f"{solver} step {k} python engine")
    e1.rheology = BINGHAM
    l0, l1 = e0.launch_count(), e1.launch_count()
    e0.step(); e1.step()
    assert e1.launch_count() - l1 > e0.launch_count() - l0, "a rheology runs the solve"
    for x in (a, c, e0, e1):
        x.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_step_graph_with_a_rheology(pkg, built, solver):
    _gpu()
    g, p = TIV._app(pkg, solver), TIV._app(pkg, solver)
    p.set_option(3, 0)
    schedule = [BINGHAM] * 4 + [None] * 2 + [CROSS] * 3
    for k, spec in enumerate(schedule):
        g.set_rheology(spec); p.set_rheology(spec)
        g.step(); p.step()
        _same(g.download(), p.download(), f"{solver} step {k}: graph vs plain launches")
        assert g.rheology_stats() == p.rheology_stats()
    assert np.array_equal(bits(g.download_viscosity()), bits(p.download_viscosity()))
    assert g.step_graph_active() and not p.step_graph_active()
    g.close(); p.close()


# ---- 7. the layers agree ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_layers_agree(pkg, built, tmp_path, solver):
    """facade, python engine and sph_headless --rheology --no-slip give the same bits over 3 frames"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    spec = dict(CROSS, beta=1.0)
    sc = pkg.scene.benchmark_scene("mini", solver)
    app, off = TIV._app(pkg, solver), TIV._app(pkg, solver)
    app.set_rheology(spec)
    s = engine.SphkSystem(sc)
    s.rheology = spec
    for k in range(3):
        app.step(); s.step(); off.step()
        a = app.download()
        _same(a, s.state(), f"{solver} frame {k}: facade vs python engine")
        assert app.rheology_stats() == s.non_newtonian_stats()
        assert np.array_equal(bits(app.download_viscosity()), bits(_np(s.nu_field)[:s.fluid.n]))
    assert not np.array_equal(bits(a["vel"]), bits(off.download()["vel"])), "the solve must change the velocities"
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    prefix = str(tmp_path / "dump")
    cmd = [TIV.CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--frames", "3", "--box", str(box), "--block", str(nx), str(ny),
           str(nz), "--origin", *[repr(float(o)) for o in origin], "--dump", prefix, "--quiet",
           "--rheology", "cross:{nu0!r},{nu_inf!r},{lam!r},{m!r}".format(**spec), "--no-slip"]
    if solver != "wcsph":
        cmd += ["--iters", "4"]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    pos = np.fromfile(prefix + ".pos.f32", np.float32).reshape(-1, 3)
    den = np.fromfile(prefix + ".density.f32", np.float32)
    assert np.array_equal(bits(pos), bits(a["pos"])) and np.array_equal(bits(den), bits(a["density"])), "sph_headless"
    app.close(); off.close(); s.close()


# ---- validation -------------------------------------------------------------------------------------------------------------
def test_entries_validate_arguments(pkg, built):
    _gpu()
    import ctypes as C
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    from cpp_fluid_particles_b200.engine import _ptr
    s = engine.SphkSystem(pkg.scene.make_scene("mini", "dfsph"), step0=False)
    L, ctx, sc = s.L, s.ctx, s._s()
    work, nuf = s._rheo_buffers()
    INVALID, STATE = -1, -4
    f, i = C.c_float, C.c_int
    good = capi.rheology(BINGHAM)

    def solve(r=good, work=work, nu=nuf, beta=1.0, dt=0.004, rho0=1.0, rhob=1.4, tol=1e-4, it=10):
        return L.sphk_non_newtonian_viscosity(ctx, sc, work, nu, C.byref(r) if r is not None else None, f(beta), f(dt), f(rho0),
                                              f(rhob), f(tol), i(it))

    def bad(**kw):
        r = capi.rheology(BINGHAM)
        for k, v in kw.items():
            if k == "p":
                r.params[v[0]] = v[1]
            else:
                setattr(r, k, v)
        return r
    nan, inf = float("nan"), float("inf")
    assert solve() == 0
    for r in (None, bad(model=0), bad(model=3), bad(nu_max=inf), bad(nu_max=nan), bad(nu_min=-1.0), bad(nu_min=1.0, nu_max=0.5),
              bad(p=(0, nan)), bad(p=(5, inf)), bad(p=(1, 0.0)), bad(p=(2, -1.0)), bad(p=(3, -1.0))):
        assert solve(r=r) == INVALID
    for kw in ({"work": None}, {"nu": None}, {"nu": work}, {"work": _ptr(s.fluid.vel)}, {"nu": _ptr(s.fluid.pos)}, {"beta": -1.0},
               {"beta": nan}, {"rho0": 0.0}, {"rhob": 0.0}, {"tol": 0.0}, {"it": 0}, {"it": 1001}):
        assert solve(**kw) == INVALID, kw
    n = s.fluid.n
    gam = torch.zeros(n, dtype=torch.float32, device=s.device)
    assert L.sphk_rheology_eval(ctx, C.byref(bad(model=7)), _ptr(gam), _ptr(s.nu_field), i(n)) == INVALID
    assert L.sphk_rheology_eval(ctx, C.byref(good), _ptr(gam), _ptr(gam), i(n)) == INVALID
    L.sphk_set_active_range(ctx, i(0), i(n // 2))
    assert solve() == STATE
    assert L.sphk_shear_rate(ctx, sc, _ptr(gam), nuf, None, None, C.byref(good), f(0), f(1.0), f(1.4)) == STATE
    L.sphk_set_active_range(ctx, i(0), i(-1))
    assert solve() == 0
    s.close()
    # dynamic bodies: beta > 0 is refused, beta = 0 runs
    sc2 = pkg.scene.make_scene("mini", "dfsph")
    body = dict(TIV._plate(sc2.fluid.mean(0), v=(0, 0, 0), w=(0, 0, 0)), mass=0.01, inertia=[1e-4, 1e-4, 1e-4])
    s = engine.SphkSystem(sc2, step0=False, bodies=[body])
    work, nuf = s._rheo_buffers()
    args = (s.ctx, s._s(), work, nuf, C.byref(good))
    assert s.L.sphk_non_newtonian_viscosity(*args, f(1.0), f(0.004), f(1.0), f(1.4), f(1e-4), i(10)) == STATE
    assert s.L.sphk_non_newtonian_viscosity(*args, f(0.0), f(0.004), f(1.0), f(1.4), f(1e-4), i(10)) == 0
    s.close()


def test_facade_refuses_and_keeps_the_setting(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    app = TIV._app(pkg, "dfsph")
    assert app.rheology_stats()["iterations"] == 0
    app.set_rheology(dict(BINGHAM, max_iter=50))
    for spec in (dict(BINGHAM, nu_max=float("inf")), dict(BINGHAM, k=-1.0), dict(BINGHAM, beta=-1.0), dict(BINGHAM, max_iter=0)):
        with pytest.raises(RuntimeError):
            app.set_rheology(spec)
    app.step()
    st = app.rheology_stats()
    assert st["iterations"] >= 1 and st["nu_max"] <= BINGHAM["nu_max"]
    app.close()
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    body = dict(TIV._plate(sc.fluid.mean(0), v=(0, 0, 0), w=(0, 0, 0)), mass=0.01, inertia=[1e-4, 1e-4, 1e-4])
    app = capi.SphApp(sc, bodies=[body])
    app.set_rheology(dict(BINGHAM, beta=0.0))
    with pytest.raises(RuntimeError):
        app.set_rheology(dict(BINGHAM, beta=1.0))
    app.step()
    assert app.rheology_stats()["iterations"] >= 1
    app.close()


# ---- 8. physics -------------------------------------------------------------------------------------------------------------
def _dam(pkg, spec, steps, solver="dfsph"):
    """mini dam break with the rheology from the first step on: (state, KE per step, iterations per step, stats of the last)"""
    app = TIV._app(pkg, solver)
    if spec is not None:
        app.set_rheology(spec)
    m = app.download()["mass"].astype(np.float64)
    ke, its = [], []
    for _ in range(steps):
        app.step()
        v = app.download()["vel"].astype(np.float64)
        ke.append(0.5 * (m * (v ** 2).sum(1)).sum())
        if spec is not None:
            its.append(app.rheology_stats()["iterations"])
    st = app.download()
    st["stats"] = app.rheology_stats() if spec is not None else None
    app.close()
    return st, np.array(ke), its


def _spread(st):
    x = st["pos"][:, [0, 2]].astype(np.float64)
    return float(np.abs(x - x.mean(0)).mean())


def _bingham(tau, nu_max=2.0):
    return dict(model="hb", k=0.01, n=1.0, tau_y=tau, m_reg=100.0, nu_max=nu_max, beta=1.0, max_iter=100)


@pytest.mark.parametrize("solver", ["dfsph", "pbd"])
def test_bingham_front_recedes_as_the_yield_stress_grows(pkg, built, solver):
    _gpu()
    taus = (0.0, 0.1, 0.4, 1.6)
    spread = [_spread(_dam(pkg, _bingham(t), 40, solver)[0]) for t in taus]
    print(f"\n{solver}: mean horizontal distance from the centre after 40 steps, tau_y = {taus}: {spread}")
    assert all(a > b for a, b in zip(spread, spread[1:])), spread


def test_yield_stress_stops_the_column(pkg, built):
    """above some tau_y the column stands: kinetic energy far below the releasable potential energy, most particles at the nu_max
    clamp.  Reports that tau_y against the estimate g H / sqrt(3) (not asserted: the estimate is unmeasured)"""
    _gpu()
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    y = sc.fluid[:, 1].astype(np.float64)
    H = float(y.max() - y.min())
    m = np.full(sc.fluid.shape[0], sc.params.m0)
    pe = float((m * 9.8 * (y - y.min())).sum())
    found = None
    rows = []
    for tau in (0.1, 0.4, 1.6, 6.4):
        st, ke, its = _dam(pkg, _bingham(tau, nu_max=5.0), 40)
        frac = st["stats"]["at_nu_max"] / st["pos"].shape[0]
        rows.append((tau, float(ke[-1] / pe), frac, max(its)))
        if found is None and ke[-1] < 0.01 * pe and frac > 0.5:
            found = tau
    print("\n".join([f"\ntau_y, KE / releasable PE after 40 steps, fraction at nu_max, max PCG iterations (H = {H:.3f}):"] +
                    [f"  {r[0]:6.2f}  {r[1]:.3e}  {r[2]:.3f}  {r[3]}" for r in rows]))
    print(f"column stands from tau_y = {found}; g H / sqrt(3) = {9.8 * H / np.sqrt(3.0):.3f}")
    assert found is not None, rows


def test_shear_thinning_front_lies_between_its_newtonian_limits(pkg, built):
    _gpu()
    nu0, nu_inf = 0.3, 0.003
    thin = dict(model="cross", nu0=nu0, nu_inf=nu_inf, lam=1.0, m=1.0, nu_max=nu0, beta=1.0, max_iter=60)
    newton = lambda nu: dict(model="cross", nu0=nu, nu_inf=nu, lam=1.0, m=1.0, nu_max=nu, beta=1.0, max_iter=60)  # noqa: E731
    s_thin, s_hi, s_lo = (_spread(_dam(pkg, spec, 40)[0]) for spec in (thin, newton(nu0), newton(nu_inf)))
    print(f"\nfront after 40 steps: Newtonian nu0 {s_hi:.4f} < Cross {s_thin:.4f} < Newtonian nu_inf {s_lo:.4f}")
    assert s_hi < s_thin < s_lo


def test_iterations_against_nu_max(pkg, built):
    """reported, not asserted beyond finiteness: how the PCG iteration count of a Bingham dam break scales with nu_max"""
    _gpu()
    rows = []
    for nu_max in (0.1, 0.5, 2.0, 8.0):
        st, ke, its = _dam(pkg, dict(_bingham(0.4, nu_max), max_iter=400), 20)
        assert np.isfinite(st["pos"]).all()
        rows.append((nu_max, float(np.mean(its)), max(its)))
    print("\nnu_max, mean / max PCG iterations over 20 steps: " + "; ".join(f"{a}: {b:.1f} / {c}" for a, b, c in rows))
    assert all(r[2] < 400 for r in rows), rows


def test_open_system_and_paddle_with_a_rheology(pkg, built):
    """an emitter + sink system (its live count changes between steps) and a kinematic paddle run with a rheology: finite, the
    solve iterates, and the facade's viscosity field has the live count"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    n0 = sc.fluid.shape[0]
    em = {"origin": (0.25, 0.40, 0.25), "direction": (0.0, -1.0, 0.0), "speed": 1.0, "spacing": 0.02, "width": 5, "height": 4}
    sinks = [((0.0, 0.0, 0.0), (0.15, 0.05, 0.15))]
    apps = [capi.SphApp(sc, max_fluid=n0 + 800, emitters=[em], sinks=sinks),
            capi.SphApp(sc, bodies=[TIV._plate(sc.fluid.mean(0), v=(0.0, 0.0, 0.0), w=(0.0, 8.0, 0.0))])]
    for app in apps:
        app.set_rheology(dict(BINGHAM, beta=0.0 if app is apps[0] else 1.0))
        counts = set()
        for _ in range(12):
            app.step()
            counts.add(app.fluid_count)
        st = app.download()
        assert np.isfinite(st["vel"]).all() and app.rheology_stats()["iterations"] >= 1
        assert app.download_viscosity().shape[0] == st["pos"].shape[0]
        if app is apps[0]:
            assert len(counts) > 1, "the live count did not change"
        app.close()


# ---- 9. sph_headless --rheology with blocking launches -------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["sph", "dfsph", "pbd"])
@pytest.mark.parametrize("extra", [[], ["--stir", "6"], ["--tap", "0.5", "--drain", "0.1"]])
def test_headless_runs_cleanly(built, tmp_path, solver, extra):
    _gpu()
    cmd = [TIV.CLI, "--solver", solver, "--frames", "3", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055",
           "0.135", "--rheology", "hb:0.02,1,0.3,100", "--rheology-max", "0.5", "--no-slip"] + \
          (["--iters", "2"] if solver != "sph" else []) + extra
    env = dict(os.environ, SPHK_STEP_GRAPH="0", CUDA_LAUNCH_BLOCKING="1")
    prefix = str(tmp_path / "dump")
    r = subprocess.run(cmd + ["--dump", prefix], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-4000:]
    bad = [line for line in r.stdout.splitlines() if "failed" in line or "error" in line.lower()]
    assert not bad, "\n".join(bad[-20:])
    assert sum("rheology" in line for line in r.stdout.splitlines()) == 3
    pos = np.fromfile(prefix + ".pos.f32", np.float32)
    assert pos.size > 0 and np.isfinite(pos).all()
