"""Kinematic rigid bodies on the GPU (DESIGN.md section 2.3): off means off, a resting body is a static boundary, placement
and pose update against the float64 reference (tests/kinematic_ref.py), the carrying boundary search, the DFSPH error
sweeps with boundary velocities on every execution path, the layers and the step graph, the physics of a rotating paddle,
and sph_headless --stir under the sanitizer's conditions."""
import dataclasses
import os
import shutil
import subprocess

import numpy as np
import pytest

import kinematic_ref as KR
import ref64
import sweep_driver as SD
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
MINI = ["--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055", "0.135"]


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _np(t):
    return t.detach().cpu().numpy().copy()


def _cli_solver(solver):
    return {"wcsph": "sph"}.get(solver, solver)


def _body(points, position, orientation=(0.0, 0.0, 0.0, 1.0), v=(0.0, 0.0, 0.0), w=(0.0, 0.0, 0.0)):
    return {"points": np.asarray(points, F), "position": [float(x) for x in position], "orientation": [float(x) for x in orientation],
            "linear_velocity": [float(x) for x in v], "angular_velocity": [float(x) for x in w]}


def _stir_scene(pkg, tmp_path, solver, omega, extra=MINI):
    """the scene of sph_headless --stir OMEGA (its --emit-scene files): (Scene, [paddle body])"""
    prefix = str(tmp_path / f"stir_{solver}_{omega}")
    r = subprocess.run([CLI, "--stir", repr(float(omega)), *extra, "--emit-scene", prefix], stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    sc = pkg.scene.benchmark_scene("mini", solver)
    box = float(extra[extra.index("--box") + 1])
    if box != float(sc.params.space[0]):
        sc = dataclasses.replace(sc, params=pkg.scene.default_params(box, solver, sc.params.dt, sc.params.max_iter,
                                                                     sc.params.density_error_threshold,
                                                                     sc.params.divergence_error_threshold))
    fluid = np.fromfile(prefix + ".fluid.f32", F).reshape(-1, 3)
    boundary = np.fromfile(prefix + ".boundary.f32", F).reshape(-1, 3)
    st = np.fromfile(prefix + ".body_state.f32", F)
    body = _body(np.fromfile(prefix + ".body.f32", F).reshape(-1, 3), st[:3], st[3:7], st[7:10], st[10:13])
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(fluid), boundary=np.ascontiguousarray(boundary)), [body]


def _same(a, b, what, fields=("pos", "vel", "density")):
    for f in fields:
        assert np.array_equal(bits(a[f]), bits(b[f])), f"{what}: {f} differs"


# ---- 1. off means off ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_no_bodies_is_the_existing_constructor(pkg, built, solver):
    """the bodies constructor with an empty vector: the same bits and the same launches per step as the existing one"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", solver)
    a, b = capi.SphApp(sc), capi.SphApp(sc, bodies=[])
    e0, e1 = engine.SphkSystem(sc), engine.SphkSystem(sc, bodies=[])
    for k in range(4):
        a.step(); b.step()
        l0, l1 = e0.launch_count(), e1.launch_count()
        e0.step(); e1.step()
        assert e0.launch_count() - l0 == e1.launch_count() - l1, f"{solver} step {k}: launches differ"
        ra = a.download()
        _same(ra, b.download(), f"{solver} step {k}: facade, empty body list")
        _same(e0.state(), e1.state(), f"{solver} step {k}: python engine, empty body list")
        assert np.array_equal(bits(a.download_boundary()["mass"]), bits(b.download_boundary()["mass"]))
    for x in (a, b, e0, e1):
        x.close()


# ---- 2. a resting body is a static boundary ---------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_resting_body_is_a_static_boundary(pkg, built, tmp_path, solver):
    """a paddle at rest (V = Omega = 0, identity pose) inside the fluid, clear of the walls by more than R, gives the bits of
    the same points, fp32(c + r), given as static boundary: placement, sort order, masses and records in one check"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc, (body,) = _stir_scene(pkg, tmp_path, solver, 0.0)
    pts = (np.asarray(body["position"], F) + body["points"]).astype(F)
    assert pts.min() > sc.params.radius + 0.01 and pts.max() < sc.params.space[0] - sc.params.radius - 0.01
    static = dataclasses.replace(sc, boundary=np.ascontiguousarray(np.concatenate([sc.boundary, pts])))
    a, b = capi.SphApp(sc, bodies=[body]), capi.SphApp(static)
    try:
        for k in range(5):
            _same(a.download(), b.download(), f"{solver} step {k}: resting body vs static points")
            ba, bb = a.download_boundary(), b.download_boundary()
            for f in ("pos", "mass"):
                assert np.array_equal(bits(ba[f]), bits(bb[f])), f"{solver} step {k}: boundary {f}"
            # particle2cell is left in pre-search order (Q2): the body run searched its boundary again from the sorted order
            assert np.array_equal(ba["p2c"], np.sort(bb["p2c"], kind="stable")), f"{solver} step {k}: boundary keys"
            a.step(); b.step()
        assert np.array_equal(a.body_pose(0), np.array([*body["position"], 0, 0, 0, 1], F))
    finally:
        a.close(); b.close()


# ---- 3. placement and pose update -------------------------------------------------------------------------------------------
def _three_bodies(rng):
    slab = np.stack(np.meshgrid((np.arange(5) - 2.0) * 0.02, (np.arange(4) - 1.5) * 0.02, [-0.01, 0.01], indexing="ij"), -1)
    slab = slab.reshape(-1, 3).astype(F)
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    return [_body(slab, (0.12, 0.3, 0.12), w=(0.0, 4.0, 0.0)),                                  # about y
            _body(slab, (0.36, 0.35, 0.36), q, v=(0.05, -0.02, 0.01), w=(1.5, -2.0, 3.0)),       # off-axis, moving
            _body(slab[::2] * F(1.5), (0.25, 0.12, 0.38), v=(0.1, 0.0, -0.05))]                  # translation only


def _ulps(x, ref, scale, what, n=8):
    tol = n * np.spacing(F(scale)).astype(np.float64)
    err = np.abs(np.asarray(x, np.float64) - ref).max()
    assert err <= tol, f"{what}: {err:.3e} > {n} ulp of {scale:.3g} ({tol:.3e})"
    return err


def test_placement_and_pose_follow_the_float64_update(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    bodies = _three_bodies(np.random.default_rng(2))
    s = engine.SphkSystem(sc, bodies=bodies, step0=False)
    dt = s.p.dt
    try:
        for k in range(12):
            if k == 6:                  # a motion change between steps takes effect at the next step
                s.set_body_motion(0, (0.0, 0.0, 0.02), (0.5, 3.0, -1.0))
            prev = s.body_pose().astype(np.float64)
            s.step()
            pose = s.body_pose()
            loc = _np(s.body_local())
            pos, vel = _np(s.boundary.pos), _np(s.boundary.vel)
            for b in range(len(bodies)):
                ref = KR.pose_update(prev[b], s.body_motion[b], np.float64(F(dt)))
                _ulps(pose[b, :3], ref[:3], np.abs(ref[:3]).max(), f"step {k} body {b} centre", 2)
                _ulps(pose[b, 3:], ref[3:], 1.0, f"step {k} body {b} quaternion", 2)
                mine = loc[:, 3] == b + 1
                assert mine.sum() == len(bodies[b]["points"])
                x, v = KR.place(pose[b].astype(np.float64), s.body_motion[b].astype(np.float64), loc[mine, :3])
                c = np.abs(pose[b, :3]).max()
                rmax = np.abs(loc[mine, :3]).max() * np.sqrt(3)
                _ulps(pos[mine], x, c + rmax, f"step {k} body {b} positions")
                m = s.body_motion[b].astype(np.float64)
                _ulps(vel[mine], v, np.abs(m[:3]).max() + np.linalg.norm(m[3:]) * rmax + 1e-30, f"step {k} body {b} velocities", 16)
            static = loc[:, 3] == 0
            assert np.all(vel[static] == 0.0)
        # drift of the orientation over many steps: body 0 now spins at constant Omega; compare with one rotation by |Omega| N dt
        q0 = s.body_pose()[0].astype(np.float64)
        N = 200
        for _ in range(N):
            s.bodies_step()
        q1 = s.body_pose()[0].astype(np.float64)
        W = s.body_motion[0, 3:].astype(np.float64)
        w = np.linalg.norm(W)
        h = 0.5 * w * N * float(F(dt))
        exact = KR.quat_mul(np.concatenate([np.sin(h) * W / w, [np.cos(h)]]), q0[3:])
        drift = np.abs(q1[3:] - exact).max()
        print(f"\norientation after {N} steps at |Omega| = {w:.3f}: max |q - q_exact| = {drift:.2e}, | |q| - 1 | = "
              f"{abs(np.linalg.norm(q1[3:]) - 1):.2e}")
        assert drift < 1e-5
    finally:
        s.close()


# ---- 4. the carrying boundary search ------------------------------------------------------------------------------------------
def test_boundary_search_carries_mass_and_body_frame(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    from oracle import oracle as O
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    bodies = _three_bodies(np.random.default_rng(5))
    # a resting body that overlaps the first one: each sums over its own particles only
    bodies.append(_body(bodies[0]["points"], (0.13, 0.31, 0.12)))
    s = engine.SphkSystem(sc, bodies=bodies, step0=False)
    plain = engine.SphkSystem(sc, step0=False)
    p = sc.params
    g = O.grid(p.cell_size, p.cell_length, hash_rcp=s.device_rcp(p.cell_length))
    try:
        # static masses: bit-identical to a run without bodies, in the same relative order
        loc = _np(s.body_local())
        static = loc[:, 3] == 0
        assert np.array_equal(bits(_np(s.boundary.mass)[static]), bits(_np(plain.boundary.mass)))
        assert np.array_equal(bits(_np(s.boundary.pos)[static]), bits(_np(plain.boundary.pos)))

        def canon(l, m):
            order = np.lexsort((l[:, 2], l[:, 1], l[:, 0], l[:, 3]))
            return m[order]

        body_mass0 = canon(loc, _np(s.boundary.mass))[static.sum():]
        for k in range(6):
            loc0, mass0, pos0 = _np(s.body_local()), _np(s.boundary.mass), _np(s.boundary.pos)
            s.step()
            st = s.state()
            loc1, mass1, pos1 = _np(s.body_local()), st["massB"], st["posB"]
            keys_pre = st["p2cB"]
            perm = np.argsort(keys_pre, kind="stable")
            assert np.array_equal(bits(loc1), bits(loc0[perm])), f"step {k}: {{r, group}} did not follow its particle"
            assert np.array_equal(bits(mass1), bits(mass0[perm])), f"step {k}: mass did not follow its particle"
            st0 = loc0[perm, 3] == 0
            assert np.array_equal(bits(pos1[st0]), bits(pos0[perm][st0])), f"step {k}: static positions moved"
            keys = O.map_cells(pos1, g)
            assert np.array_equal(keys, keys_pre[perm]), f"step {k}: sorted keys"
            assert np.all(np.diff(keys) >= 0)
            cs = np.searchsorted(keys, np.arange(p.ncells + 1), side="left").astype(np.int32)
            assert np.array_equal(cs, st["cell_startB"]), f"step {k}: cell_start of the boundary set"
            assert np.array_equal(bits(canon(loc1, mass1)[static.sum():]), bits(body_mass0)), f"step {k}: body masses changed"
        # grouped masses against the float64 reference (a body sees only itself, the static set only itself); they are
        # invariant under rigid motion, so the reference at the last positions is the one at construction
        ref = KR.grouped_masses(pos1, loc1[:, 3], p.rho_boundary, p.radius)
        assert np.abs(mass1 - ref).max() <= 1e-5 * ref.max()
        overlap = np.isin(loc1[:, 3], [1, 4])
        whole = KR.grouped_masses(pos1, np.zeros(len(pos1)), p.rho_boundary, p.radius)
        assert np.abs(whole - ref)[overlap].max() > 1e-2 * ref.max(), "the overlapping bodies must test the grouping"
    finally:
        s.close(); plain.close()


# ---- 5. the DFSPH error sweeps with boundary velocities on every path ---------------------------------------------------------
def _paddle_case(pkg):
    """jittered mini block with a paddle (rotating about an off-vertical axis and translating) in its middle"""
    sc = pkg.scene.make_scene("mini", solver="dfsph", jitter=0.003, max_iter=4, den_thr=-1.0, div_thr=-1.0)
    slab = np.stack(np.meshgrid((np.arange(6) - 2.5) * 0.0198, (np.arange(10) - 4.5) * 0.0198, [-0.0099, 0.0099], indexing="ij"), -1)
    c = sc.fluid.mean(0)
    d = sc.fluid - c
    keep = ~((np.abs(d[:, 0]) < 0.07) & (np.abs(d[:, 1]) < 0.11) & (np.abs(d[:, 2]) < 0.03))
    fluid = np.ascontiguousarray(sc.fluid[keep])
    body = _body(slab.reshape(-1, 3), c, v=(0.2, -0.1, 0.05), w=(1.0, 6.0, -2.0))
    return dataclasses.replace(sc, fluid=fluid), [body]


def _error_setup(pkg, scene, path, bodies_override=None):
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    if scene == "walls":
        sc, bodies = SD.make_case(pkg, "walls").sc, None
    else:
        sc, bodies = _paddle_case(pkg)
    if bodies_override is not None:
        bodies = bodies_override(bodies)
    s = engine.SphkSystem(sc, step0=False, use_list=path.use_list, list_capacity=path.kmax, bodies=bodies)
    s.set_option(capi.OPT_STAGED_LIST_BUILD, path.staged)
    s.set_option(capi.OPT_TILE, path.tile)
    s.set_use_list(path.use_list, path.skin)
    return s, sc, torch


@pytest.mark.parametrize("path", sorted(SD.PATHS))
@pytest.mark.parametrize("scene", ["walls", "paddle"])
def test_dfsph_errors_with_boundary_velocities(pkg, built, scene, path):
    _gpu()
    from oracle import oracle as O
    s, sc, torch = _error_setup(pkg, scene, SD.PATHS[path])
    p = sc.params
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))   # noqa: E731
    try:
        if s.n_bodies:
            s.bodies_step()                    # the paddle has moved once: positions off its initial lattice, velocities set
        s.search_fluid()
        st = s.state()
        n = s.fluid.n
        g = O.grid(p.cell_size, p.cell_length, hash_rcp=s.device_rcp(p.cell_length))
        A = O.SceneArrays(st["pos"], st["mass"], st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius)
        P = ref64.Pairs(A)
        velB = _np(s.boundary.vel)
        if s.n_bodies:
            assert np.abs(velB).max() > 0.1 and len(P.iB) > 0
        vel = (0.5 * np.sin(7.0 * st["pos"]) + 0.05 * np.random.default_rng(7).standard_normal((n, 3))).astype(F)

        def set_vel(v):             # the fluid search packs the fluid records; the boundary records are the body search's
            s.fluid.vel.copy_(t(v))
            s.search_fluid()

        s.dfsph_density_alpha()
        dens, alpha = s.state()["density"], _np(s.alpha)
        for label, refresh_only in (("", False), (" after sphk_refresh", True)):
            set_vel(vel)
            if refresh_only:         # sphk_refresh must keep the body velocities in the boundary records (then a search
                s.refresh()          # again: the sweeps take this case's path, not the cell walk of a refreshed set)
                s.search_fluid()
            s.fluid.density.copy_(t(dens)); s.alpha.copy_(t(alpha))
            s.dfsph_div_error()
            re_, rk = KR.dfsph_div_error(P, vel, velB, dens, alpha, p.dt, p.rho0, ref64.TAU)
            ref64.assert_per_element(_np(s.error), re_, ref64.TAU, f"{scene}/{path} divergence error{label}")
            ref64.assert_per_element(_np(s.kappa), rk, ref64.TAU, f"{scene}/{path} divergence stiffness{label}")
            set_vel(vel)
            if refresh_only:
                s.refresh()
                s.search_fluid()
            dens_hi = (dens * F(1.28)).astype(F)
            s.fluid.density.copy_(t(dens_hi)); s.alpha.copy_(t(alpha))
            s.warm.zero_()
            s.dfsph_den_error(False)
            re_, rk = KR.dfsph_den_error(P, vel, velB, dens_hi, alpha, p.dt, p.rho0)
            ref64.assert_per_element(_np(s.error), re_, ref64.TAU, f"{scene}/{path} density error{label}", re_.floor)
            ref64.assert_per_element(_np(s.kappa), rk, ref64.TAU, f"{scene}/{path} density stiffness{label}", rk.floor)
    finally:
        s.close()


@pytest.mark.parametrize("path", ["cells", "list", "tile", "skin"])
def test_galilean_motion_has_zero_divergence_error(pkg, built, path):
    """fluid and body all moving at V, Omega = 0: the divergence error is exactly 0 and the density error is the one at rest"""
    _gpu()
    V = np.array([0.3, -0.2, 0.4], F)

    def translate(bodies):
        return [dict(b, linear_velocity=[float(x) for x in V], angular_velocity=[0.0, 0.0, 0.0]) for b in bodies]

    s, sc, torch = _error_setup(pkg, "paddle", SD.PATHS[path], translate)
    p = sc.params
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))   # noqa: E731
    try:
        s.bodies_step()
        s.search_fluid()
        n = s.fluid.n
        mine = _np(s.body_local())[:, 3] > 0
        assert np.array_equal(bits(_np(s.boundary.vel)[mine]), bits(np.tile(V, (int(mine.sum()), 1)))), "v_k = V for Omega = 0"
        s.dfsph_density_alpha()
        dens = (s.state()["density"] * F(1.1)).astype(F)
        out = {}
        for label, v in (("moving", np.tile(V, (n, 1))), ("rest", None)):
            if v is None:            # everything at rest (the refresh below packs the zeroed body velocities)
                s.boundary.vel.zero_()
                v = np.zeros((n, 3), F)
            s.fluid.vel.copy_(t(v))
            s.refresh()
            s.fluid.density.copy_(t(dens))
            s.dfsph_div_error()
            out[label + "_div"] = _np(s.error)
            s.fluid.density.copy_(t(dens))
            s.dfsph_den_error(False)
            out[label + "_den"] = _np(s.error)
        assert np.all(out["moving_div"] == 0.0), f"{path}: divergence error of a Galilean motion"
        assert np.array_equal(bits(out["moving_den"]), bits(out["rest_den"])), f"{path}: density error of a Galilean motion"
        assert out["rest_den"].max() > 0
    finally:
        s.close()


# ---- 6. layers and graph -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", SOLVERS)
def test_layers_agree_with_a_paddle(pkg, built, tmp_path, solver):
    """class layer (facade), python engine and sph_headless --stir give the same bits over 3 frames"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    omega = 4.0
    sc, bodies = _stir_scene(pkg, tmp_path, solver, omega)
    app = capi.SphApp(sc, bodies=bodies)
    s = engine.SphkSystem(sc, bodies=bodies)
    try:
        for k in range(3):
            app.step(); s.step()
            a = app.download()
            _same(a, s.state(), f"{solver} frame {k}: facade vs python engine", ("pos", "density"))
            assert np.array_equal(app.body_pose(0), s.body_pose()[0])
        assert np.array_equal(bits(app.download_boundary()["pos"]), bits(s.state()["posB"]))
        prefix = str(tmp_path / "dump")
        cmd = [CLI, "--solver", _cli_solver(solver), "--frames", "3", *MINI, "--dump", prefix, "--quiet", "--stir", repr(omega)]
        if solver != "wcsph":
            cmd += ["--iters", "4"]
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        pos = np.fromfile(prefix + ".pos.f32", F).reshape(-1, 3)
        den = np.fromfile(prefix + ".density.f32", F)
        assert np.array_equal(bits(pos), bits(a["pos"])) and np.array_equal(bits(den), bits(a["density"])), "sph_headless --stir"
    finally:
        app.close(); s.close()
    bad = subprocess.run([CLI, "--stir", "2", "--ranks", "2", "--frames", "0"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert bad.returncode != 0 and "--stir" in bad.stderr


@pytest.mark.parametrize("solver", SOLVERS)
def test_step_graph_with_motion_changes(pkg, built, tmp_path, solver):
    """graph on and off agree bit for bit while the motion changes between steps, and a motion change keeps the graph"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc, bodies = _stir_scene(pkg, tmp_path, solver, 3.0)
    g, p = capi.SphApp(sc, bodies=bodies), capi.SphApp(sc, bodies=bodies)
    p.set_option(3, 0)
    schedule = [((0, 0, 0), (0, 3, 0))] * 3 + [((0.05, 0, 0), (0, -2, 0))] * 2 + [((0, 0, 0), (1, 0, 0.5))] * 3
    try:
        for k, (v, w) in enumerate(schedule):
            had = g.step_graph_active()
            g.set_body_motion(0, v, w); p.set_body_motion(0, v, w)
            if had:
                assert g.step_graph_active(), f"{solver} step {k}: a motion change dropped the step graph"
            g.step(); p.step()
            _same(g.download(), p.download(), f"{solver} step {k}: graph vs plain launches")
            assert np.array_equal(g.body_pose(0), p.body_pose(0))
        assert g.step_graph_active() and not p.step_graph_active()
    finally:
        g.close(); p.close()


def test_body_arguments_are_validated(pkg, built):
    _gpu()
    import ctypes as C
    from cpp_fluid_particles_b200 import capi, engine
    from cpp_fluid_particles_b200 import slabs
    L = capi.sphk()
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s = engine.SphkSystem(sc, step0=False)
    fp = lambda a: np.ascontiguousarray(a, F).ctypes.data_as(C.POINTER(C.c_float))   # noqa: E731
    try:
        b = s.boundary.abi()
        n = s.boundary.n
        # bodies after the first boundary search, and steps without bodies: call order
        begin = (C.c_int * 2)(n - 4, n)
        assert L.sphk_bodies_init(s.ctx, C.byref(b), n - 4, 1, begin, fp(np.zeros(12)), fp([0, 0, 0, 0, 0, 0, 1]), fp(np.zeros(6))) == -4
        assert L.sphk_bodies_step(s.ctx, C.byref(b), C.c_void_p(s.cs_boundary.data_ptr()), C.c_float(0.004)) == -4
        assert L.sphk_bodies_set_motion(s.ctx, fp(np.zeros(6))) == -4
    finally:
        s.close()
    with pytest.raises(ValueError):
        slabs.SlabSystem(sc, 0, 1, "cuda:0", bodies=[_body(np.zeros((1, 3)), (0.2, 0.2, 0.2))])
    # invalid arguments on a fresh context
    from cpp_fluid_particles_b200.capi import SphkGrid
    import torch
    g = SphkGrid()
    g.cell_size[:] = [int(c) for c in sc.params.cell_size]
    g.cell_length = sc.params.cell_length
    ctx = C.c_void_p()
    capi.check(L.sphk_create(C.byref(ctx), C.c_int(100), C.c_int(200), C.byref(g), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    try:
        pos = torch.zeros((200, 3), device="cuda")
        vel, mass = torch.zeros_like(pos), torch.zeros(200, device="cuda")
        p2c = torch.zeros(200, dtype=torch.int32, device="cuda")
        pa = capi.SphkParticles()
        pa.pos, pa.vel, pa.mass, pa.particle2cell, pa.n = pos.data_ptr(), vel.data_ptr(), mass.data_ptr(), p2c.data_ptr(), 200
        ok_begin = (C.c_int * 3)(100, 150, 200)
        loc, pose, mot = np.zeros(300), np.tile([0.2, 0.2, 0.2, 0, 0, 0, 1], 2), np.zeros(12)

        def init(begin=ok_begin, nb=2, pose=pose, mot=mot, loc=loc, n_static=100, null=None):
            args = [ctx, C.byref(pa), n_static, nb, begin, fp(loc), fp(pose), fp(mot)]
            if null is not None:
                args[null] = None
            return L.sphk_bodies_init(*args)

        assert init(null=1) == -1 and init(null=4) == -1 and init(null=5) == -1 and init(null=6) == -1 and init(null=7) == -1
        assert init(begin=(C.c_int * 3)(100, 160, 150)) == -1, "non-monotonic body_begin"
        assert init(begin=(C.c_int * 3)(90, 150, 200)) == -1, "body_begin[0] != n_static"
        assert init(nb=65, begin=(C.c_int * 66)(*([100] * 65 + [200]))) == -1, "more than 64 bodies"
        assert init(pose=np.tile([0.2, np.nan, 0.2, 0, 0, 0, 1], 2)) == -1 and init(mot=np.array([np.inf] + [0] * 11)) == -1
        assert init(pose=np.tile([0.2, 0.2, 0.2, 0, 0, 0, 0], 2)) == -1, "zero quaternion"
        pa.vel = None
        assert init() == -1, "boundary velocities are needed"
        pa.vel = vel.data_ptr()
        cs = torch.zeros(sc.params.ncells + 1, dtype=torch.int32, device="cuda")
        assert L.sphk_bodies_step(ctx, C.byref(pa), C.c_void_p(cs.data_ptr()), C.c_float(0.004)) == -4, "step before init"
        assert init() == 0
        assert L.sphk_bodies_step(ctx, C.byref(pa), C.c_void_p(cs.data_ptr()), C.c_float(0.004)) == -4, "step before the first search"
        capi.check(L.sphk_neighbor_search(ctx, 1, C.byref(pa), C.c_void_p(cs.data_ptr())))
        for dt in (0.0, -0.004, float("nan"), float("inf")):
            assert L.sphk_bodies_step(ctx, C.byref(pa), C.c_void_p(cs.data_ptr()), C.c_float(dt)) == -1, dt
        assert L.sphk_bodies_step(ctx, C.byref(pa), None, C.c_float(0.004)) == -1
        assert L.sphk_bodies_set_motion(ctx, fp(np.array([np.nan] + [0] * 11))) == -1
        assert L.sphk_bodies_set_motion(ctx, None) == -1 and L.sphk_bodies_get_pose(ctx, None) == -1
        assert L.sphk_bodies_step(ctx, C.byref(pa), C.c_void_p(cs.data_ptr()), C.c_float(0.004)) == 0
        assert init() == -4, "a second init"
        capi.check(L.sphk_synchronize(ctx))
    finally:
        L.sphk_destroy(ctx)


# ---- 7. physics: a paddle stirring fluid at rest ------------------------------------------------------------------------------
# a block that covers the floor of the 0.5 box (at rest under gravity up to the lattice's settling), paddle through its middle
POOL = ["--box", "0.5", "--block", "23", "12", "23", "--origin", "0.03", "0.03", "0.03"]


@pytest.mark.parametrize("solver", SOLVERS)
def test_rotating_paddle_stirs_the_fluid(pkg, built, tmp_path, solver):
    """after 60 steps the fluid's angular momentum about the paddle axis has the sign of Omega (both signs), and no fluid
    particle is inside the paddle's slab within its extent.  With -s the numbers are printed (DESIGN.md section 2.3)."""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    steps = 60
    for omega in (5.0, -5.0):
        sc, (body,) = _stir_scene(pkg, tmp_path, solver, omega, POOL)
        s = engine.SphkSystem(sc, bodies=[body])
        try:
            for _ in range(steps):
                s.step()
            st = s.state()
            pose = s.body_pose()[0].astype(np.float64)
        finally:
            s.close()
        c = pose[:3]
        d = st["pos"].astype(np.float64) - c
        v = st["vel"].astype(np.float64)
        m = st["mass"].astype(np.float64)
        Ly = (m * (d[:, 2] * v[:, 0] - d[:, 0] * v[:, 2])).sum()
        pts = body["points"].astype(np.float64)
        hw, hh, ht = np.abs(pts).max(0)
        ref = abs(omega) * (m * (d[:, 0] ** 2 + d[:, 2] ** 2) * ((d[:, 0] ** 2 + d[:, 2] ** 2) < hw * hw)).sum()
        local = d @ KR.rotation(pose[3:])                      # body-frame coordinates R^T d
        inside = (np.abs(local[:, 2]) < ht) & (np.abs(local[:, 0]) < hw) & (np.abs(local[:, 1]) < hh)
        print(f"\n[{solver}] Omega {omega:+.1f} rad/s, {steps} steps: L_y = {Ly:.3e}, L_y / (|Omega| I_swept) = {Ly / ref:+.3f}, "
              f"paddle turned {2 * np.degrees(np.arctan2(np.linalg.norm(pose[3:6]), pose[6])):.1f} deg, inside the slab: {int(inside.sum())}")
        # measured on an H100: L_y / (|Omega| I_swept) = 0.63 (WCSPH, dt 0.001), 1.60 (DFSPH), 1.24 (PBD), both signs
        assert np.sign(Ly) == np.sign(omega) and abs(Ly) > 0.3 * ref, f"{solver} Omega {omega}: L_y = {Ly:.3e} (swept {ref:.3e})"
        assert not inside.any(), f"{solver}: {int(inside.sum())} fluid particles inside the paddle"


# ---- 8. sanitizer -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["sph", "dfsph", "pbd"])
def test_stir_memcheck(built, tmp_path, solver):
    """sph_headless --stir as test_gpu_sanitizer runs its apps: blocking launches, plain steps, clean exit and finite particles;
    under compute-sanitizer memcheck with SPHK_SANITIZER=1"""
    cmd = [CLI, "--solver", solver, "--frames", "3", *MINI, "--quiet", "--stir", "4"]
    if solver != "sph":
        cmd += ["--iters", "2"]
    env = dict(os.environ, SPHK_STEP_GRAPH="0")
    if os.environ.get("SPHK_SANITIZER") == "1":
        exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
        assert os.path.exists(exe), "SPHK_SANITIZER=1 but compute-sanitizer is not installed"
        r = subprocess.run([exe, "--tool", "memcheck", "--error-exitcode", "9"] + cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=900, env=env)
        assert r.returncode == 0 and "ERROR SUMMARY: 0 errors" in r.stdout, r.stdout[-4000:]
        return
    prefix = str(tmp_path / "dump")
    env["CUDA_LAUNCH_BLOCKING"] = "1"
    r = subprocess.run(cmd + ["--dump", prefix], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-4000:]
    bad = [line for line in r.stdout.splitlines() if "failed" in line or "error" in line.lower()]
    assert not bad, "\n".join(bad[-20:])
    pos = np.fromfile(prefix + ".pos.f32", F)
    den = np.fromfile(prefix + ".density.f32", F)
    assert pos.size == 3 * den.size > 0 and np.isfinite(pos).all() and np.isfinite(den).all()
