"""The engine's reductions beyond one block (DESIGN.md section 2.7): the abs-sum of the DFSPH error and the device loop test
bit for bit against the float32 emulation of their fixed shape (tests/reduction_ref.py), adaptive DFSPH at 2M particles, the
implicit-viscosity dot products at 2M, body impulses past one block of 256 particles, all 64 body poses, and the fluid mass
range of the search and of sphk_refresh at 2M."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

import implicit_visc_ref as IV
import kinematic_ref as KR
import reduction_ref as RD
import ref64
import rigid_ref as RR
from test_gpu_rigid import _body, _check_reaction, _cube
from util import bits

pytestmark = pytest.mark.gpu

F = np.float32
CAP = 1024 * 2048                       # elements past which the first stage strides past its 1024 blocks


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _np(t):
    return t.detach().cpu().numpy().copy()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, F)).cuda()


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _mixed(n, seed, denormals=False):
    """seeded mixed-sign values spread over 2^+-20 (and, with denormals, every 5th one below 2^-126)"""
    rng = np.random.default_rng(seed)
    x = (rng.choice([-1.0, 1.0], n) * np.exp2(rng.uniform(-20, 20, n))).astype(F)
    if denormals:
        x[::5] = (rng.choice([-1.0, 1.0], x[::5].size) * rng.uniform(1e-45, 1.1e-38, x[::5].size)).astype(F)
    return x


@pytest.fixture(scope="module")
def mini(pkg, built):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    s = engine.SphkSystem(pkg.scene.make_scene("mini"), step0=False)
    yield s
    s.close()


# ---- 1. the abs-sum, direct -------------------------------------------------------------------------------------------------
SIZES = [1, 31, 255, 256, 2047, 2048, 2049, 256 * 2048 - 1, 256 * 2048 + 1, 257 * 2048, CAP - 1, CAP + 1, 3 * 2 ** 21 + 7]


def _loop_total(s, x_dev, n):
    """one device-loop iteration over x: the total k_loop_finish stores"""
    L = s.L
    assert L.sphk_loop_begin(s.ctx, 0, 1, 1, C.c_float(0.0), 1) == 0
    assert L.sphk_loop_next(s.ctx, 0, _ptr(x_dev), n) == 0
    assert L.sphk_loop_end(s.ctx, 0) == 0
    it, tot = C.c_int(0), C.c_float(0.0)
    assert L.sphk_loop_iterations(s.ctx, 0, C.byref(it), C.byref(tot)) == 0
    assert it.value == 1
    return F(tot.value)


@pytest.mark.parametrize("n,denormals", [(n, False) for n in SIZES] + [(2049, True), (CAP + 1, True)])
def test_abs_sum_is_the_fixed_shape_bit_for_bit(mini, n, denormals):
    x = _mixed(n, 1000 + n, denormals)
    xd = _dev(x)
    out = C.c_float(0.0)
    assert mini.L.sphk_reduce_abs_sum(mini.ctx, _ptr(xd), n, C.byref(out)) == 0
    got, ref = F(out.value), RD.tree_abs_sum(x)
    assert bits(np.array([got]))[0] == bits(np.array([ref]))[0], f"n = {n}: {got!r} vs the emulation {ref!r}"
    exact = RD.exact_abs_sum(x)
    assert abs(float(got) - exact) <= RD.bound(x), f"n = {n}: |sum - fsum| = {abs(float(got) - exact):.3e}"
    loop = _loop_total(mini, xd, n)
    assert bits(np.array([loop]))[0] == bits(np.array([got]))[0], f"n = {n}: device-loop total {loop!r} vs {got!r}"
    print(f"\nn = {n}: |x - fsum| / sum|x| = {abs(float(got) - exact) / exact:.2e} (bound {RD.bound(x) / exact:.2e})")


# ---- 2. loop control, direct ------------------------------------------------------------------------------------------------
N_SMALL = 4096
T = F(4.0)                               # N_SMALL x 2^-10: arrays of powers of two give exact totals


def _flat(v, n=N_SMALL, last=None):
    a = np.full(n, v, F)
    if last is not None:
        a[-1] = last
    return a


ARRAYS = {
    "big": _flat(2.0 ** -6),                                        # total 64
    "equal": _flat(2.0 ** -10),                                     # exactly T
    "above": _flat(2.0 ** -10, last=2.0 ** -10 + 2.0 ** -21),       # T + 1 ulp
    "below": _flat(2.0 ** -10, last=2.0 ** -10 - 2.0 ** -22),       # T - 1 ulp
    "small": _flat(2.0 ** -14),
    "huge": _flat(1.0e30),
    "nan": _flat(2.0 ** -10, last=np.nan),
}
CASES = {   # name: (min_iter, max_iter, reduce_from, arrays)
    "stops at the threshold": (1, 20, 1, ["big", "big", "equal", "big"]),
    "one ulp above": (1, 20, 1, ["big", "above", "below", "big"]),
    "one ulp below": (1, 20, 1, ["big", "big", "below", "big"]),
    "reduce_from 2, huge first": (2, 20, 2, ["huge", "small", "big"]),
    "min_iter 2, small first": (2, 20, 1, ["small", "big", "small", "big"]),
    "max_iter 0": (1, 0, 1, ["big", "big"]),
    "max_iter 1": (1, 1, 1, ["big", "big"]),
    "max_iter 20": (1, 20, 1, ["big"] * 22),
    "nan": (1, 20, 1, ["big", "nan", "big", "big"]),
}


def _run_loop(s, arrays, min_iter, max_iter, thr, reduce_from, n, before=None):
    L = s.L
    assert L.sphk_loop_begin(s.ctx, 1, min_iter, max_iter, C.c_float(thr), reduce_from) == 0
    for a in arrays:
        if before is not None:
            before()
        assert L.sphk_loop_next(s.ctx, 1, _ptr(a), n) == 0
    assert L.sphk_loop_end(s.ctx, 1) == 0
    it, tot = C.c_int(0), C.c_float(0.0)
    assert L.sphk_loop_iterations(s.ctx, 1, C.byref(it), C.byref(tot)) == 0
    return it.value, F(tot.value)


def _same_loop(got, ref, what):
    assert got[0] == ref[0], f"{what}: {got[0]} iterations, the model {ref[0]}"
    if np.isnan(ref[1]):                 # (the device's NaN is the canonical one, not the payload of the input)
        assert np.isnan(got[1]), f"{what}: last total {got[1]!r}, the model NaN"
        return
    assert bits(np.array([got[1]]))[0] == bits(np.array([ref[1]]))[0], f"{what}: last total {got[1]!r}, the model {ref[1]!r}"


@pytest.mark.parametrize("case", sorted(CASES))
def test_loop_control_follows_the_model(mini, case):
    min_iter, max_iter, rf, names = CASES[case]
    host = [ARRAYS[k] for k in names]
    totals = [RD.tree_abs_sum(a) for a in host]
    exact = {"equal": T, "above": np.nextafter(T, F(np.inf)), "below": np.nextafter(T, F(0))}
    for k, t in zip(names, totals):      # the crafted totals are exact
        assert k not in exact or t == exact[k], k
    got = _run_loop(mini, [_dev(a) for a in host], min_iter, max_iter, T, rf, N_SMALL)
    _same_loop(got, RD.loop_model(min_iter, max_iter, T, rf, totals), case)


@pytest.mark.parametrize("n", [257 * 2048 + 3, CAP + 2049])
def test_loop_control_at_scale(mini, n):
    """past 256 partials and past the 1024-block cap: thresholds just below, at and above the second total"""
    x = np.abs(_mixed(n, n))
    host = [x * F(4), x * F(2), x, x * F(0.5)]
    totals = [RD.tree_abs_sum(a) for a in host]
    dev = [_dev(a) for a in host]
    for thr in (np.nextafter(totals[1], F(0)), totals[1], np.nextafter(totals[1], F(np.inf)), totals[2]):
        got = _run_loop(mini, dev, 1, 20, thr, 1, n)
        _same_loop(got, RD.loop_model(1, 20, thr, 1, totals), f"n = {n}, threshold {thr!r}")


def test_converged_loop_gates_the_sweeps(pkg, built):
    """DFSPH divergence corrections enqueued once per iteration, as DFSPHSolver does: converged at iteration 3 of 5, the
    velocities equal a run with max_iter = 3 bit for bit (the corrections after convergence return at once).  The fluid
    starts with seeded random velocities, so that every correction changes them."""
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    sc = _squeezed(pkg.scene.make_scene("mini", solver="dfsph", dt=0.004))
    v0 = np.random.default_rng(9).uniform(-0.5, 0.5, (sc.n_fluid, 3)).astype(F)
    converging = ("big", "big", "below", "big", "big")
    vel = {}
    for name, max_iter, names, iters in (("converged", 5, converging, 3), ("max 3", 3, converging, 3), ("max 4", 4, ("big",) * 5, 4)):
        s = engine.SphkSystem(sc, step0=False)
        try:
            s.fluid.vel.copy_(torch.from_numpy(v0).cuda())
            s.search_fluid()
            s.dfsph_density_alpha()
            s.dfsph_div_error()
            dev = [_dev(ARRAYS[k]) for k in names]
            assert _run_loop(s, dev, 1, max_iter, T, 1, N_SMALL, before=s.dfsph_div_correct)[0] == iters, name
            vel[name] = _np(s.fluid.vel)
        finally:
            s.close()
    assert np.array_equal(bits(vel["converged"]), bits(vel["max 3"])), "a correction ran after the loop converged"
    assert not np.array_equal(bits(vel["max 4"]), bits(vel["max 3"])), "one more correction changes nothing: the check would be empty"


# ---- 3. adaptive DFSPH at 2M --------------------------------------------------------------------------------------------------
def _squeezed(sc, f=0.9):
    """the fluid block shrunk about its centre: denser than rho0, so that the DFSPH errors are not clamped to 0 from the start"""
    c = sc.fluid.mean(0, dtype=np.float64)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray((c + f * (sc.fluid - c)).astype(F)))


def _scene_2m(pkg, extra):
    sc = _squeezed(pkg.scene.make_scene("2m", solver="dfsph", dt=0.004, den_thr=1e-3, div_thr=1e-3, max_iter=20))
    if extra:                            # a block in a free corner: n = 2^21 + 2049, past the 1024-block cap
        a = np.arange(13, dtype=F) * F(0.02)
        blk = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)[:extra] + F(0.1)
        sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(np.concatenate([sc.fluid, blk.astype(F)])))
    return sc


@pytest.mark.parametrize("extra", [0, 2049])
def test_adaptive_dfsph_2m_device_and_host_loops(pkg, built, extra):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = _scene_2m(pkg, extra)
    dev, host = capi.SphApp(sc), capi.SphApp(sc)
    host.set_option(1, 0)
    try:
        for k in range(4):
            dev.step(); host.step()
            it = dev.dfsph_iterations()
            assert it == host.dfsph_iterations(), f"step {k}: device {it} vs host {host.dfsph_iterations()}"
            a, b = dev.download(), host.download()
            for f in ("pos", "vel", "density"):
                assert np.array_equal(bits(a[f]), bits(b[f])), f"step {k}: {f}"
        print(f"\n2m + {extra}: last step's iterations {it}")
        assert it[0] < 20 or it[1] < 20, "no loop converged: the test never decided on a sum"
    finally:
        dev.close(); host.close()


@pytest.mark.parametrize("extra", [0, 2049])
def test_adaptive_dfsph_2m_host_sums_and_decisions(pkg, built, extra):
    """every error sum of the host loop equals the emulation bit for bit; each continue / stop decision equals the float64
    decision wherever |fsum - threshold| exceeds the bound"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = _scene_2m(pkg, extra)
    s = engine.SphkSystem(sc)
    n = s.fluid.n
    thr = s.den_thr * n * s.p.rho0
    assert s.div_thr == s.den_thr
    orig = s.reduce_abs_sum
    seen = {"calls": 0, "nonzero": 0, "decided": 0, "worst": 0.0}

    def checked(x):
        got = orig(x)
        a = _np(x)
        assert a.size == n
        ref = RD.tree_abs_sum(a)
        assert bits(np.array([F(got)]))[0] == bits(np.array([ref]))[0], f"call {seen['calls']}: {got!r} vs {ref!r}"
        exact, b = RD.exact_abs_sum(a), RD.bound(a)
        if exact > 0:
            seen["nonzero"] += 1
            seen["worst"] = max(seen["worst"], abs(got - exact) / exact)
        if abs(exact - thr) > b:
            assert (got > thr) == (exact > thr), f"call {seen['calls']}: sum {got!r}, fsum {exact!r}, threshold {thr!r}"
            seen["decided"] += 1
        seen["calls"] += 1
        return got

    s.reduce_abs_sum = checked
    try:
        for _ in range(4):
            s.step()
    finally:
        s.close()
    print(f"\n2m + {extra}: {seen['calls']} sums ({seen['nonzero']} non-zero), {seen['decided']} decisions checked, "
          f"largest |x - fsum| / sum = {seen['worst']:.2e}")
    assert seen["nonzero"] >= 4 and seen["decided"] >= 4


# ---- 4. implicit viscosity at 2M -----------------------------------------------------------------------------------------------
HEAD = 64
PARTS = 1024


def _head(work):
    raw = _np(work[:HEAD]).view(np.uint8)
    ints = raw[:16].view(np.int32)
    d = raw[16:64].view(np.float64)
    return {"active": int(ints[0]), "iters": int(ints[1]), "max_iter": int(ints[2]), "tol2": d[0], "bb": d[1], "rz": d[2],
            "rr": d[3], "alpha": d[4], "beta": d[5]}


def _mdot(m, a, b):
    """sum_i m_i a_i . b_i with its float64 rounding bound: 64 * 2^-53 * sum |terms|"""
    t = np.asarray(m, np.float64) * (np.asarray(a, np.float64) * np.asarray(b, np.float64)).sum(1)
    return math.fsum(t.tolist()), 64 * 2.0 ** -53 * float(np.abs(t).sum())


@pytest.mark.parametrize("extra", [0, 2049])
def test_implicit_viscosity_dot_products_2m(pkg, built, extra):
    _gpu()
    import torch
    from cpp_fluid_particles_b200 import engine
    sc = _scene_2m(pkg, extra)
    s = engine.SphkSystem(sc, step0=False)
    n = s.fluid.n
    nu = 0.1
    try:
        assert s.L.sphk_implicit_viscosity_work_floats(C.c_int(n)) == 6208 + 21 * n
        rng = np.random.default_rng(7)
        v0 = torch.from_numpy(rng.uniform(-0.5, 0.5, (n, 3)).astype(F)).cuda()
        s.fluid.vel[:n].copy_(v0)
        s.search_fluid()                 # the records carry the velocities (permuted with the particles)
        x0 = _np(s.fluid.vel[:n])
        mass = _np(s.fluid.mass[:n])
        for max_iter in (1, 2, 3):
            s.fluid.vel[:n].copy_(torch.from_numpy(x0).cuda())
            s.refresh()
            D = torch.zeros((n, 6), dtype=torch.float32, device="cuda")
            b = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
            Ax0 = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
            s.visc_implicit_setup(D, b, nu, nu)
            s.visc_implicit_matvec(D, s.fluid.vel[:n], Ax0, nu)
            s.fluid.vel[:n].copy_(torch.from_numpy(x0).cuda())
            s.refresh()
            s.implicit_viscosity(nu=nu, nu_boundary=nu, tol=1e-12, max_iter=max_iter)
            it, res = s.implicit_viscosity_stats()
            h = _head(s.visc_work)
            assert it == max_iter == h["iters"], (it, h)
            w = s.visc_work
            off = HEAD + 2 * 3 * PARTS
            r = _np(w[off + 12 * n: off + 15 * n]).reshape(n, 3)
            bb, bb_tol = _mdot(mass, _np(b), _np(b))
            rr, rr_tol = _mdot(mass, r, r)
            assert abs(h["bb"] - bb) <= bb_tol, f"max_iter {max_iter}: <b,b> {h['bb']!r} vs {bb!r}"
            assert abs(h["rr"] - rr) <= rr_tol, f"max_iter {max_iter}: <r,r> {h['rr']!r} vs {rr!r}"
            assert res == float(F(np.sqrt(h["rr"] / h["bb"]))), (res, h)
            print(f"\n2m + {extra}, max_iter {max_iter}: |bb - fsum| / tol = {abs(h['bb'] - bb) / bb_tol:.2f}, "
                  f"|rr - fsum| / tol = {abs(h['rr'] - rr) / rr_tol:.2f}, residual {res:.3e}")
            if max_iter != 1:
                continue
            # the step of the first iteration: alpha = <r0, z0>_M / <z0, A z0>_M
            Dinv = _np(w[off + 6 * n: off + 12 * n]).reshape(n, 6)
            r0 = (_np(b) - _np(Ax0)).astype(F)
            z0 = np.einsum("nab,nb->na", IV.unpacked(Dinv), r0.astype(np.float64))
            Az0 = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
            s.visc_implicit_matvec(D, torch.from_numpy(z0.astype(F)).cuda(), Az0, nu)
            rz, _ = _mdot(mass, r0, z0)
            zAz, _ = _mdot(mass, z0, _np(Az0))
            alpha = rz / zAz
            assert abs(h["alpha"] - alpha) <= 1e-5 * abs(alpha), f"alpha {h['alpha']!r} vs {alpha!r}"
            x1 = _np(s.fluid.vel[:n]).astype(np.float64)
            step = h["alpha"] * z0
            tol = 4 * np.spacing(np.abs(x1).astype(F)).astype(np.float64) + 1e-5 * np.abs(step)
            assert (np.abs(x1 - x0 - step) <= tol).all(), "x1 - x0 is not alpha z0"
    finally:
        s.close()


# ---- 5. bodies beyond one block -----------------------------------------------------------------------------------------------
def _trimmed(k):
    p = _cube(8)                         # 296 particles
    return p[296 - k:]


def test_body_impulses_past_one_block(pkg, built):
    """bodies of 255, 256, 257, 296 and 728 particles and an empty one: {J, H} against the float64 pair sums after a reacting
    divergence correction, and the end-of-step update against rigid_ref.integrate"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    from test_gpu_rigid import _params
    sc = _params(pkg, "dfsph")
    rng = np.random.default_rng(3)
    fluid = sc.fluid + rng.uniform(-0.15, 0.15, sc.fluid.shape).astype(F) * F(0.02)
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(fluid.astype(F)))
    q = np.array([0.3, -0.5, 0.2, 0.8]); q /= np.linalg.norm(q)
    bodies = [_body(_trimmed(255), (0.2, 0.15, 0.2), v=(0.1, 0.0, 0.0), rel=1.0),
              _body(_trimmed(256), (0.27, 0.2, 0.27), w=(1.0, -2.0, 0.5), q=q, rel=0.8),
              _body(_trimmed(257), (0.22, 0.25, 0.28), v=(0.0, -0.1, 0.05), rel=1.2),
              _body(np.zeros((0, 3), F), (0.3, 0.3, 0.3), v=(0.05, 0.02, -0.01)),
              _body(_cube(8), (0.25, 0.18, 0.22), w=(0.0, 0.5, 0.0), rel=1.0),
              _body(_cube(12), (0.24, 0.2, 0.24), v=(0.0, 0.0, 0.1), rel=0.9)]
    bodies[3]["mass"], bodies[3]["inertia"] = 1e-3, [1e-7, 1e-7, 1e-7]
    sizes = [len(b["points"]) for b in bodies]
    assert sizes == [255, 256, 257, 0, 296, 728]
    s = engine.SphkSystem(sc, bodies=bodies, step0=False)
    dt = float(F(sc.params.dt))
    G = np.array(sc.params.gravity, np.float64)
    try:
        s.bodies_step()
        s.search_fluid()
        s.dfsph_density_alpha(); s.dfsph_div_error(); s.dfsph_div_correct()
        s.bodies_react(1.0)
        before = s.current_body_motion().astype(np.float64)
        _check_reaction(s, len(bodies), _np(s.fluid.pos), _np(s.kappa), 1.0, "bodies past one block")
        JH = s.body_impulse()
        got = s.current_body_motion().astype(np.float64)
        pose = s.body_pose().astype(np.float64)
        for b, body in enumerate(bodies):
            ref = RR.integrate(before[b], pose[b, 3:], body["mass"], body["inertia"], JH[b, :3].astype(np.float64),
                               JH[b, 3:].astype(np.float64), dt, G)
            tol = 1e-5 * (np.abs(ref) + np.abs(before[b]) + 1e-3)
            assert (np.abs(got[b] - ref) <= tol).all(), f"body {b} ({sizes[b]} particles): {got[b]} vs {ref}"
        assert not JH[3].any(), f"the empty body gathered {JH[3]}"
        assert np.array_equal(got[3, :3].astype(F), (before[3, :3] + dt * G).astype(F)) and not got[3, 3:].any()
    finally:
        s.close()


def test_all_64_poses_follow_the_float64_update(pkg, built):
    """SPHK_MAX_BODIES kinematic bodies, each with its own motion: every pose after each of 3 body steps against
    kinematic_ref.pose_update, body 63 included"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    rng = np.random.default_rng(64)
    g = (np.arange(4) + 0.5) * 0.1 + 0.05
    centres = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    bodies = []
    for c in centres:
        qq = rng.standard_normal(4); qq /= np.linalg.norm(qq)
        bodies.append(_body(_cube(2), c, v=rng.uniform(-0.2, 0.2, 3), w=rng.uniform(-3, 3, 3), q=qq))
    assert len(bodies) == 64
    s = engine.SphkSystem(sc, bodies=bodies, step0=False)
    dt = np.float64(F(sc.params.dt))
    try:
        for k in range(3):
            prev = s.body_pose().astype(np.float64)
            s.bodies_step()
            pose = s.body_pose().astype(np.float64)
            for b in range(64):
                ref = KR.pose_update(prev[b], s.body_motion[b], dt)
                assert np.abs(pose[b, :3] - ref[:3]).max() <= 2 * np.spacing(F(np.abs(ref[:3]).max())), f"step {k} body {b}"
                assert np.abs(pose[b, 3:] - ref[3:]).max() <= 2 * np.spacing(F(1.0)), f"step {k} body {b} quaternion"
    finally:
        s.close()


# ---- 6. the fluid mass range at 2M --------------------------------------------------------------------------------------------
def _density_near(s, slot, what):
    """the density of the particle in `slot` and of its fluid neighbours against ref64.density over that neighbourhood"""
    s.set_use_list(False)
    s.density()
    st = s.state()
    x, m = st["pos"].astype(np.float64), st["mass"].astype(np.float64)
    R = float(s.p.radius)
    c = x[slot]
    near = np.flatnonzero((np.abs(x - c) <= 3 * R).all(1))
    xb, mb = st["posB"].astype(np.float64), st["massB"].astype(np.float64)
    nearB = np.flatnonzero((np.abs(xb - c) <= 3 * R).all(1))
    targets = np.flatnonzero(np.linalg.norm(x[near] - c, axis=1) <= R)
    assert targets.size > 10 and slot in near[targets]

    class A:                               # the neighbourhood as one in-grid cell range
        posF, massF, posB, massB = x[near], m[near], xb[nearB], mb[nearB]
        csF, csB = np.array([near.size]), np.array([nearB.size])
        g = type("G", (), {"ncells": 0})
    A.R = R
    ref = ref64.density(ref64.Pairs(A))
    sub = dataclasses.replace(ref, value=ref.value[targets], mag=ref.mag[targets])
    ref64.assert_per_element(st["density"][near[targets]], sub, ref64.TAU, what)
    uniform = ref64.density(ref64.Pairs(A, masses=np.full(near.size, float(s.p.m0))))
    miss = np.abs(uniform.value[targets] - ref.value[targets])
    assert (miss[near[targets] != slot] > 100 * ref64.TAU * ref.mag[targets][near[targets] != slot]).any(), \
        "the heavy particle does not show in its neighbours' density: the check would be empty"


@pytest.mark.parametrize("where", ["last slot, search", "middle slot, refresh"])
def test_mass_range_2m(pkg, built, where):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.benchmark_scene("2m", "dfsph")
    s = engine.SphkSystem(sc, step0=False)
    n = s.fluid.n
    m0 = F(s.p.m0)
    try:
        slot = n - 1 if where.startswith("last") else n // 2 + 12345
        s.fluid.mass[slot] = float(F(4) * m0)
        if where.startswith("last"):
            s.search_fluid()             # masses stay in their slots (Q2): the search packs slot n - 1's mass
        else:
            s.refresh()
        _density_near(s, slot, where)
    finally:
        s.close()
