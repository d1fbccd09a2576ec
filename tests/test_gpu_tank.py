"""Tank motion on the GPU (DESIGN.md section 2.15): sphk_tank_force per element against the float64 reference (tests/tank_ref.py),
the device per-step state and frame time, no change when off or zero, graph and plain steps, the Coriolis rotation, the physics of
a tilted surface, a spinning bucket and a resonant roll on the 23 x 12 x 23 pool with gauges for all three solvers, and the
combinations with dynamic bodies, checkpoints, CFL steps, open boundaries and the headless app."""
import ctypes as C
import dataclasses
import json
import os
import subprocess

import numpy as np
import pytest

import rigid_ref as RR
import tank_ref as TR
from util import ROOT, bits

pytestmark = pytest.mark.gpu

F = np.float32
SOLVERS = ["wcsph", "dfsph", "pbd"]
CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
SPACING = 0.02
M0 = 76.596750762082e-6
RHO_MASS = M0 / SPACING ** 3
EPS32 = 2.0 ** -24

ROLL = dict(axis=(0.0, 0.0, 1.0), pivot=(0.25, 0.0, 0.25), roll_amplitude=0.2, roll_omega=5.0, roll_phase=0.4, ramp=0.6)
SPIN = dict(axis=(0.0, 1.0, 0.0), pivot=(0.25, 0.0, 0.25), spin=3.0, ramp=0.6)
SHAKE = dict(accel=(1.5, 0.0, 0.0), harmonics=[dict(amplitude=(3.0, 0.0, 1.0), omega=9.0), dict(amplitude=(0.0, 2.0, 0.0), omega=4.0,
                                                                                                  phase=0.5)], ramp=0.6)


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _np(t):
    return t.detach().cpu().numpy().copy()


def _same(a, b, what, fields=("pos", "vel", "density")):
    for f in fields:
        assert np.array_equal(bits(a[f]), bits(b[f])), f"{what}: {f} differs"


def _eval(L, spec, G, t):
    from cpp_fluid_particles_b200 import capi
    out = (C.c_float * capi.TANK_STATE)()
    assert L.sphk_tank_eval(C.byref(capi.tank_motion(spec)), (C.c_float * 3)(*G), C.c_double(t), out) == 0
    return np.array(out[:], np.float32)


# ---- 1. per element ---------------------------------------------------------------------------------------------------------------
def _jittered(pkg, seed=5):
    import torch
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    rng = np.random.default_rng(seed)
    fl = (sc.fluid + rng.uniform(-0.2, 0.2, sc.fluid.shape).astype(F) * SPACING).astype(F)
    s = engine.SphkSystem(dataclasses.replace(sc, fluid=np.ascontiguousarray(fl)), step0=False)
    n = s.fluid.n
    s.fluid.vel[:n] = torch.from_numpy(rng.uniform(-0.5, 0.5, (n, 3)).astype(F)).to(s.device)
    s.refresh()
    return s


@pytest.mark.parametrize("name,spec", [("roll", ROLL), ("spin", SPIN), ("shake", SHAKE)])
def test_force_matches_float64_per_element(pkg, built, name, spec):
    """one sphk_tank_force at t on both sides of the ramp's end against tank_ref.step: a few float ulps of the sum of the terms'
    magnitudes; the device state within one float ulp of sphk_tank_eval and the frame time advanced by (double) dt"""
    _gpu()
    s = _jittered(pkg)
    L, G = s.L, tuple(float(F(g)) for g in s.p.gravity)
    dt = float(F(s.p.dt))
    try:
        s.tank = spec
        n = s.fluid.n
        x, v0 = _np(s.fluid.pos)[:n], _np(s.fluid.vel)[:n]
        for t in (0.05, 0.59, 0.61, 1.3):
            assert L.sphk_tank_set_time(s.ctx, C.c_double(t)) == 0
            s.tank_force(dt)
            got = _np(s.fluid.vel)[:n].astype(np.float64)
            ref, terms = TR.step(spec, G, t, dt, x, v0)
            mag = sum(np.abs(v) for v in terms.values())
            err = np.abs(got - ref)
            assert (err <= 6 * EPS32 * mag + 1e-12).all(), f"{name} t={t}: worst {(err / (mag + 1e-30)).max() / EPS32:.2f} ulps"
            moved = np.abs(ref - v0).max()
            assert moved > 100 * err.max(), f"{name} t={t}: the step does not change v measurably"
            td, st = s.tank_state()
            assert td == t + dt, (td, t + dt)
            e = _eval(L, spec, G, t)
            assert (np.abs(st - e) <= np.spacing(np.abs(e))).all(), f"{name} t={t}: device state {st} vs {e}"
            s.fluid.vel[:n] = s.fluid.vel.new_tensor(v0)
            s.refresh()
    finally:
        s.close()


def test_context_refusals_change_nothing(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    s = _jittered(pkg)
    L, G = s.L, (C.c_float * 3)(*[float(g) for g in s.p.gravity])
    try:
        assert L.sphk_tank_force(s.ctx, s._s(), C.c_float(0.004)) == -4             # no motion yet
        assert L.sphk_tank_time(s.ctx, C.byref(C.c_double()), None) == -4
        assert L.sphk_tank_set_time(s.ctx, C.c_double(0.0)) == -4
        s.tank = ROLL
        for bad in (dict(axis=(0.0, 0.0, 0.0)), dict(roll_omega=-1.0), dict(ramp=np.nan)):
            assert L.sphk_tank_set(s.ctx, C.byref(capi.tank_motion(bad)), G) == -1
        for t in (-1.0, np.nan, np.inf):
            assert L.sphk_tank_set_time(s.ctx, C.c_double(t)) == -1
        for dt in (-0.001, np.nan):
            assert L.sphk_tank_force(s.ctx, s._s(), C.c_float(dt)) == -1
        assert L.sphk_set_active_range(s.ctx, 0, 100) == 0
        assert L.sphk_tank_set(s.ctx, C.byref(capi.tank_motion(SPIN)), G) == -4     # slab ranks
        assert L.sphk_set_active_range(s.ctx, 0, -1) == 0
        assert s.tank_state()[0] == 0.0                   # nothing enqueued, the motion kept: the roll's state after one step
        s.tank_force()
        e = _eval(L, ROLL, [float(F(g)) for g in s.p.gravity], 0.0)
        assert (np.abs(s.tank_state()[1] - e) <= np.spacing(np.abs(e))).all()
    finally:
        s.close()


def test_frame_time_equals_the_simulated_time(pkg, built):
    """after N steps (the constructor's step 0 first, then the motion) the device frame time is the host's simulated time, bit for
    bit, and the facade's tank state is the schedule at that time"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s, app = engine.SphkSystem(sc, tank=ROLL), capi.SphApp(sc)
    try:
        app.set_tank_motion(ROLL)
        for _ in range(37):
            s.step(); app.step()
        td, _ = s.tank_state()
        assert td == s.simulated_time
        ts = app.tank_state()
        assert ts["t"] == s.simulated_time
        e = _eval(s.L, ROLL, [float(F(g)) for g in sc.params.gravity], ts["t"])
        assert [ts["theta"], ts["theta_dot"], ts["theta_ddot"]] == list(e[:3])
        assert np.array_equal(ts["gravity"], e[3:6]) and np.array_equal(ts["accel"], e[6:9])
        _same(app.download(), s.state(), "facade vs python engine, rolled")
    finally:
        s.close(); app.close()


# ---- 2. no change when off or zero ------------------------------------------------------------------------------------------------
ZERO = dict(axis=(0.3, 0.0, 1.0), pivot=(0.25, 0.0, 0.25), roll_omega=5.0, harmonics=[dict(amplitude=(0.0, 0.0, 0.0), omega=3.0)],
            ramp=0.1)


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_motion_and_a_cleared_motion_change_nothing(pkg, built, solver):
    """every amplitude zero: particles bit-identical to the system without a motion over 20 steps (graph steps); a motion set and
    cleared again: the same bits and the same launches per step"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", solver)
    off, zero = capi.SphApp(sc), capi.SphApp(sc)
    e_off, e_clr = engine.SphkSystem(sc), engine.SphkSystem(sc, tank=ROLL)
    try:
        zero.set_tank_motion(ZERO)
        e_clr.tank = None
        for k in range(20):
            off.step(); zero.step()
            n0 = e_off.launch_count()
            e_off.step()
            n1 = e_clr.launch_count()
            e_clr.step()
            assert e_clr.launch_count() - n1 == e_off.launch_count() - n0
            _same(off.download(), zero.download(), f"{solver} step {k}: zero motion", ("pos", "vel", "density", "pressure"))
            _same(e_off.state(), e_clr.state(), f"{solver} step {k}: cleared motion", ("pos", "vel", "density", "pressure"))
        assert off.step_graph_active() and zero.step_graph_active()
    finally:
        off.close(); zero.close(); e_off.close(); e_clr.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_graph_and_plain_steps_agree_with_a_rolling_tank(pkg, built, solver):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", solver)
    g, p, still = capi.SphApp(sc), capi.SphApp(sc), capi.SphApp(sc)
    try:
        p.set_option(3, 0)
        for a in (g, p):
            a.set_tank_motion(ROLL)
        for k in range(20):
            g.step(); p.step(); still.step()
            _same(g.download(), p.download(), f"{solver} step {k}: graph vs plain")
        assert g.step_graph_active() and not p.step_graph_active()
        assert not np.array_equal(bits(g.download()["vel"]), bits(still.download()["vel"])), "the motion must change the flow"
    finally:
        g.close(); p.close(); still.close()


# ---- 3. Coriolis ------------------------------------------------------------------------------------------------------------------
def test_coriolis_keeps_the_speed(pkg, built):
    """spin only, gravity off, particles on the spin axis (the Euler and centrifugal terms vanish exactly): 1000 sphk_tank_force
    calls rotate every v about the axis and keep |v|.  The rotation is done in double; what remains is the float rounding of v
    at every call, a random walk: the median drift stays below 1e-6, the worst of 512 particles below 4e-6 (DESIGN.md section
    2.15), and the mean signed drift shows no growth -- an explicit -2 Omega x v kick would grow |v| by 33 % here."""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    rng = np.random.default_rng(11)
    n = 512
    y = 0.03 + 0.4 * np.arange(n) / n
    fl = np.stack([np.full(n, 0.25), y, np.full(n, 0.25)], 1).astype(F)
    s = engine.SphkSystem(dataclasses.replace(sc, fluid=np.ascontiguousarray(fl)), step0=False)
    try:
        v0 = rng.uniform(-1.0, 1.0, (n, 3)).astype(F)
        s.fluid.vel[:n] = torch.from_numpy(v0).to(s.device)
        s.refresh()
        spin = dict(axis=(0.0, 1.0, 0.0), pivot=(0.25, 0.0, 0.25), spin=3.0)
        assert s.L.sphk_tank_set(s.ctx, C.byref(capi.tank_motion(spin)), (C.c_float * 3)(0.0, 0.0, 0.0)) == 0
        dt = 0.004
        for _ in range(1000):
            s.tank_force(dt)
        v = _np(s.fluid.vel)[:n].astype(np.float64)
        r = np.linalg.norm(v, axis=1) / np.linalg.norm(v0.astype(np.float64), axis=1) - 1.0
        print(f"\ncoriolis: |v| drift after 1000 calls: median {np.median(np.abs(r)):.2e}, max {np.abs(r).max():.2e}, "
              f"mean {r.mean():.2e}")
        assert np.median(np.abs(r)) <= 1e-6 and np.abs(r).max() <= 4e-6 and abs(r.mean()) <= 3e-7
        assert np.array_equal(v[:, 1], v0[:, 1].astype(np.float64)), "the axial component is untouched"
        ang = np.arctan2(v[:, 0], v[:, 2]) - np.arctan2(v0[:, 0], v0[:, 2])
        expect = -2.0 * 3.0 * float(F(dt)) * 1000           # Rot(n, -2 Omega dt) per call
        d = np.angle(np.exp(1j * (ang - expect)))
        assert np.abs(d).max() < 1e-3, "v turned by -2 Omega t about the axis"
    finally:
        s.close()


# ---- 4. physics on the pool -------------------------------------------------------------------------------------------------------
C0 = 0.2475                                   # the centre of the clamp box [0, 0.99 * 0.5]


def _pool(pkg, solver):
    sc = pkg.scene.benchmark_scene("mini", solver)
    a, b = np.arange(23) * SPACING, np.arange(12) * SPACING
    fl = np.stack(np.meshgrid(a, b, a, indexing="ij"), -1).reshape(-1, 3) + 0.03
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(fl.astype(F)))


def _gauge(x, z):
    return ((x, 0.002, z), (x, 0.48, z), 240)


def _levels(pkg, solver, motion, gauges, seconds):
    """the gauges' levels after every step of `seconds` of the pool under `motion` (facade, step graph), and the step times"""
    from cpp_fluid_particles_b200 import capi
    sc = _pool(pkg, solver)
    steps = int(round(seconds / float(F(sc.params.dt))))
    app = capi.SphApp(sc)
    try:
        app.set_tank_motion(motion)
        app.set_probes([], gauges, capacity=steps)
        for _ in range(steps):
            app.step()
        s = app.probe_series()
        assert np.isfinite(app.download()["pos"]).all()
        return s["times"], s["levels"]
    finally:
        app.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_tilted_surface(pkg, built, solver):
    """a constant a_c = 4 m/s^2 along x, ramped over 1.5 s: the surface settles at the slope |a_c| / |G| (Delta h over the gauges
    0.38 m apart: 0.155 m, about 8 spacings), averaged over the last 0.8 s, within 20 %"""
    _gpu()
    a, g = 4.0, 9.8
    t, lv = _levels(pkg, solver, dict(accel=(a, 0.0, 0.0), ramp=1.5), [_gauge(0.055, C0), _gauge(0.435, C0)], 3.0)
    late = t > t[-1] - 0.8
    slope = (lv[late, 0].mean() - lv[late, 1].mean()) / 0.38
    print(f"\n[{solver}] tilted surface: slope {slope:.4f}, expected {a / g:.4f} (ratio {slope / (a / g):.3f})")
    assert abs(slope / (a / g) - 1.0) <= 0.2


@pytest.mark.parametrize("solver", SOLVERS)
def test_spinning_bucket(pkg, built, solver):
    """spin Omega0 = 6.5 rad/s about the vertical axis through the centre, ramped over 1.5 s: the level at r = 0.24 (a diagonal)
    above the centre's by Omega0^2 r^2 / (2 |G|) = 0.125 m (6 spacings), averaged over the last 1.5 s of 6 s, within 20 %"""
    _gpu()
    W, g, d = 6.5, 9.8, 0.17
    spin = dict(axis=(0.0, 1.0, 0.0), pivot=(C0, 0.0, C0), spin=W, ramp=1.5)
    t, lv = _levels(pkg, solver, spin, [_gauge(C0, C0), _gauge(C0 + d, C0 + d)], 6.0)
    late = t > t[-1] - 1.5
    dh = lv[late, 1].mean() - lv[late, 0].mean()
    ref = W * W * 2 * d * d / (2 * g)
    print(f"\n[{solver}] spinning bucket: rim - centre {dh:.4f} m, expected {ref:.4f} (ratio {dh / ref:.3f})")
    assert abs(dh / ref - 1.0) <= 0.2


@pytest.mark.parametrize("solver", SOLVERS)
def test_roll_resonance(pkg, built, solver):
    """roll of 1.5 degrees about the z axis through the bottom centre at the first linear mode w1^2 = (pi |G| / L) tanh(pi h / L)
    (L = 0.495 between the walls, h = 0.207 the settled depth) and at w1 / 2: the wall gauge's range over 1.5-5 s at w1 is at
    least twice the range at w1 / 2"""
    _gpu()
    L, h, g = 0.495, 0.207, 9.8
    w1 = float(np.sqrt(np.pi * g / L * np.tanh(np.pi * h / L)))
    rng = {}
    for w in (w1, 0.5 * w1):
        roll = dict(axis=(0.0, 0.0, 1.0), pivot=(C0, 0.0, C0), roll_amplitude=float(np.radians(1.5)), roll_omega=w, ramp=0.5)
        t, lv = _levels(pkg, solver, roll, [_gauge(0.03, C0)], 5.0)
        late = t > 1.5
        rng[w] = float(np.ptp(lv[late, 0]))
    print(f"\n[{solver}] roll resonance: w1 = {w1:.3f} rad/s, wall gauge range {rng[w1]:.4f} m at w1, {rng[0.5 * w1]:.4f} m at w1/2 "
          f"(ratio {rng[w1] / rng[0.5 * w1]:.2f})")
    assert rng[w1] >= 2.0 * rng[0.5 * w1]


# ---- 5. combinations --------------------------------------------------------------------------------------------------------------
def _cube(side_pts, h=SPACING):
    a = (np.arange(side_pts) - 0.5 * (side_pts - 1)) * h
    p = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    return p[(np.abs(p) > a.max() - 1e-9).any(1)].astype(F)


def _body(points, position, rel=None):
    b = {"points": np.asarray(points, F), "position": [float(x) for x in position], "orientation": [0.0, 0.0, 0.0, 1.0],
         "linear_velocity": [0.0, 0.0, 0.0], "angular_velocity": [0.0, 0.0, 0.0]}
    if rel is not None:
        side = np.ptp(b["points"][:, 0]) + SPACING
        M = rel * RHO_MASS * side ** 3
        b["mass"], b["inertia"] = float(M), [float(M * side * side / 6)] * 3
    return b


def test_dynamic_cube_in_a_shaken_tank(pkg, built):
    """each step's integrated motion of a dynamic cube equals rigid_ref.integrate with G - a_w(t_n); a rotating motion is refused
    with dynamic bodies in every layer, and dynamics are refused under a rotating motion"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    body = _body(_cube(4), (0.25, 0.2, 0.25), rel=0.8)
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    shake = dict(accel=(1.5, 0.0, -0.5), harmonics=[dict(amplitude=(3.0, 0.0, 1.0), omega=9.0)])
    s = engine.SphkSystem(sc, bodies=[body], step0=False)
    G = [float(F(g)) for g in sc.params.gravity]
    dt = float(F(sc.params.dt))
    try:
        with pytest.raises(ValueError):
            s.tank = SPIN
        assert s.L.sphk_tank_set(s.ctx, C.byref(capi.tank_motion(ROLL)), (C.c_float * 3)(*G)) == -4
        s.tank = shake
        for k in range(6):
            before = s.current_body_motion()[0].astype(np.float64)
            tn = s.simulated_time
            s.step()
            pose = s.body_pose()[0].astype(np.float64)
            JH = s.body_impulse()[0].astype(np.float64)
            got = s.current_body_motion()[0].astype(np.float64)
            geff = TR.state(shake, G, tn)[3:6]
            ref = RR.integrate(before, pose[3:], body["mass"], body["inertia"], JH[:3], JH[3:], dt, geff)
            tol = 1e-5 * (np.abs(ref) + np.abs(before) + 1e-3)
            assert (np.abs(got - ref) <= tol).all(), f"step {k}: {got} vs {ref}"
            plain = RR.integrate(before, pose[3:], body["mass"], body["inertia"], JH[:3], JH[3:], dt, G)
            assert np.abs(got[:3] - plain[:3]).max() > 100 * tol[:3].max(), "the case does not tell G - a_w from G"
    finally:
        s.close()
    app = capi.SphApp(sc, bodies=[body])
    try:
        with pytest.raises(RuntimeError):
            app.set_tank_motion(SPIN)
        app.set_tank_motion(shake)
    finally:
        app.close()
    held = dict(body, mass=0.0, inertia=[0.0, 0.0, 0.0])
    k = engine.SphkSystem(sc, bodies=[held], step0=False)
    try:
        k.tank = SPIN                                 # rotation with a kinematic body is supported ...
        mi = np.array([[body["mass"], *body["inertia"]]], F)
        assert k.L.sphk_bodies_set_dynamics(k.ctx, mi.ctypes.data_as(C.POINTER(C.c_float)), k._space) == -4   # ... dynamics not
        k.step()
    finally:
        k.close()


@pytest.mark.parametrize("solver", SOLVERS)
def test_checkpoint_resume_with_a_rolling_tank(pkg, built, solver, tmp_path):
    """checkpoint at step 10 of a rolled run and resume in a fresh system: bit-identical to the uninterrupted run at step 25; a
    restore under another motion, or without one, is refused"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", solver)
    path = str(tmp_path / "rolled.ckpt")
    a = capi.SphApp(sc)
    try:
        a.set_tank_motion(ROLL)
        for _ in range(10):
            a.step()
        a.checkpoint(path)
        for _ in range(15):
            a.step()
        a.checkpoint_wait()
        ref = a.download()
    finally:
        a.close()
    b = capi.SphApp(sc)
    try:
        b.set_tank_motion(ROLL)
        b.restore(path)
        for _ in range(15):
            b.step()
        _same(ref, b.download(), f"{solver}: resumed vs uninterrupted", ("pos", "vel", "density", "pressure"))
    finally:
        b.close()
    for other in (dict(ROLL, roll_omega=5.5), None):
        c = capi.SphApp(sc)
        try:
            if other is not None:
                c.set_tank_motion(other)
            before = c.download()
            with pytest.raises(RuntimeError):
                c.restore(path)
            _same(before, c.download(), "a refused restore changes nothing")
        finally:
            c.close()


def test_cfl_run_of_a_hard_shake(pkg, built):
    """a 3 g shake at 8 Hz with CFL steps: the rule's |G| is sphk_tank_accel_bound (the first adaptive dt is the rule's output for
    it, and shorter than with |G|: C is small enough that the bound, not dt_max, decides it), every frame stays finite, and both
    layers' rules agree"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    hard = dict(harmonics=[dict(amplitude=(30.0, 0.0, 10.0), omega=2 * np.pi * 8)], ramp=0.05)
    app = capi.SphApp(sc)
    cfl = 0.01
    e = engine.SphkSystem(sc, adaptive=dict(C=cfl), tank=hard)
    L = e.L
    try:
        app.set_adaptive_dt(cfl)
        app.set_tank_motion(hard)
        bound = C.c_double(0.0)
        assert L.sphk_tank_accel_bound(C.byref(capi.tank_motion(hard)), e._G, e._space, C.byref(bound)) == 0
        assert e._rule.gravity == bound.value and bound.value > 30.0
        app.step()
        st = app.adaptive_stats()
        r = capi.SphkTimeStepRule()
        dtmax = float(F(sc.params.dt))
        r.cfl, r.dt_max, r.dt_min, r.radius, r.gravity = float(F(cfl)), dtmax, float(F(dtmax) / F(64)), float(F(sc.params.radius)), bound.value
        dt, flags = C.c_float(0.0), C.c_int(0)
        assert L.sphk_time_step(C.byref(r), C.c_double(st["speed"]), C.c_double(dtmax), C.c_double(0.0), C.byref(dt), C.byref(flags)) == 0
        assert st["last_dt"] == dt.value
        r.gravity = 9.8
        L.sphk_time_step(C.byref(r), C.c_double(st["speed"]), C.c_double(dtmax), C.c_double(0.0), C.byref(dt), C.byref(flags))
        assert st["last_dt"] < dt.value, "the bound must shorten the step"
        for _ in range(5):
            app.advance(0.02)
            assert np.isfinite(app.download()["vel"]).all()
        assert app.adaptive_stats()["nonfinite_steps"] == 0
    finally:
        app.close(); e.close()


def test_paddle_tap_drain_and_gauges_under_a_motion(built, tmp_path):
    """a stirring paddle, a tap, a drain and gauges in a rolled and shaken tank: the headless app runs clean and its gauges read
    finite levels"""
    _gpu()
    csv = str(tmp_path / "g.csv")
    r = subprocess.run([CLI, "--solver", "dfsph", "--iters", "4", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055",
                        "0.135", "--frames", "60", "--quiet", "--stir", "2", "--tap", "1.0", "--drain", "0.1", "--tank-roll", "4,1",
                        "--tank-shake", "1,0,0,2", "--tank-ramp", "0.05", "--gauge", "0.05,0.002,0.25,0.05,0.45,0.25,128",
                        "--gauge", "0.44,0.002,0.25,0.44,0.45,0.25,128", "--probe-out", csv],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert res["emitted"] > 0
    rows = np.loadtxt(csv, delimiter=",", skiprows=1, ndmin=2)
    assert rows.shape[0] == 60 and np.isfinite(rows).all() and (rows[:, -2:] >= -1).all() and (rows[:, -2:] > 0).any()


@pytest.mark.parametrize("solver", SOLVERS)
def test_headless_dump_agrees(pkg, built, solver, tmp_path):
    """sph_headless --tank-roll's dump, the facade and the python engine agree bit for bit, and every frame line prints theta"""
    _gpu()
    from cpp_fluid_particles_b200 import capi, engine
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["mini"]
    base = [CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--box", str(box), "--block", str(nx), str(ny), str(nz),
            "--origin", *[repr(float(o)) for o in origin]] + (["--iters", "4"] if solver != "wcsph" else [])
    prefix = str(tmp_path / "scene")
    r = subprocess.run(base + ["--quiet", "--emit-scene", prefix], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    sc = pkg.scene.benchmark_scene("mini", solver)
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(np.fromfile(prefix + ".fluid.f32", np.float32).reshape(-1, 3)))
    dump = str(tmp_path / "dump")
    r = subprocess.run(base + ["--frames", "6", "--tank-roll", "4,1.5", "--tank-ramp", "0.01", "--dump", dump], capture_output=True,
                       text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert sum("tank - theta" in ln for ln in r.stdout.splitlines()) == 6
    roll = dict(axis=(0.0, 0.0, 1.0), pivot=(0.25, 0.0, 0.25), roll_amplitude=float(F(4.0 * np.pi / 180.0)),
                roll_omega=float(F(2.0 * np.pi * 1.5)), ramp=0.01)
    app, e = capi.SphApp(sc), engine.SphkSystem(sc, tank=roll)
    try:
        app.set_tank_motion(roll)
        for _ in range(6):
            app.step(); e.step()
        a = app.download()
        _same(a, e.state(), f"{solver}: facade vs python engine")
        pos = np.fromfile(dump + ".pos.f32", np.float32).reshape(-1, 3)
        den = np.fromfile(dump + ".density.f32", np.float32)
        assert np.array_equal(bits(pos), bits(a["pos"])) and np.array_equal(bits(den), bits(a["density"])), "sph_headless"
    finally:
        app.close(); e.close()
