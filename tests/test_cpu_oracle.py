"""The CPU restatement (oracle/) against: the committed golden outputs of the reference's own CUDA
kernels (tests/golden/, generated on an H100 by tests/golden/make_golden.py), analytic values, and the
structural properties the reference's algorithm guarantees.  Runs without a GPU."""
import json
import os

import numpy as np
import pytest

from util import GOLDEN, assert_close, cell_start_from_p2c, relerr


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def _rcp_from_meta():
    path = os.path.join(GOLDEN, "meta.json")
    if not os.path.exists(path):
        return 0.0
    bits = json.load(open(path))["rcp_cell_length_bits"]
    return float(np.uint32(bits).view(np.float32))


def test_scene_counts_match_survey(pkg):
    # SURVEY.md section 8: N_f / N_b / cells of the named configurations
    for name, nf, nb, nc in (("config0", 20736, 14408, 25), ("2m", 2097152, 237608, 100)):
        sc = pkg.scene.make_scene(name)
        assert sc.fluid.shape == (nf, 3) and sc.boundary.shape == (nb, 3) and sc.params.cell_size == (nc,) * 3
        assert pkg.scene.near_face_count(sc.fluid, sc.params.cell_length) == 0
    sc = pkg.scene.make_scene("config0")
    # main.cpp:79-81: first point (0.27, 0.10, 0.27), z fastest, then x, y slowest
    assert np.allclose(sc.fluid[0], [0.27, 0.10, 0.27]) and np.isclose(sc.fluid[1, 2] - sc.fluid[0, 2], 0.02)
    assert np.isclose(sc.fluid[24, 0] - sc.fluid[0, 0], 0.02) and np.isclose(sc.fluid[24 * 24, 1] - sc.fluid[0, 1], 0.02)
    assert sc.boundary.min() >= 0.005 - 1e-7 and sc.boundary.max() <= 0.995 + 1e-6


def test_neighbor_search_properties(pkg, O):
    sc = pkg.scene.make_scene("config0", jitter=0.002)
    g = O.grid(sc.params.cell_size, sc.params.cell_length)
    vel = np.arange(sc.fluid.size, dtype=np.float32).reshape(-1, 3)
    pos_s, vel_s, p2c, cs, perm = O.neighbor_search(sc.fluid, vel, g)
    n, nc = sc.fluid.shape[0], sc.params.ncells
    assert np.array_equal(np.sort(perm), np.arange(n))
    ks = p2c[perm]
    assert np.all(np.diff(ks) >= 0)
    assert np.all(np.diff(perm)[np.diff(ks) == 0] > 0), "stable"
    assert np.array_equal(pos_s, sc.fluid[perm]) and np.array_equal(vel_s, vel[perm])
    assert np.array_equal(cs, cell_start_from_p2c(p2c, nc)) and cs[-1] == n
    # idempotence
    pos2, _, p2c2, cs2, perm2 = O.neighbor_search(pos_s, vel_s, g)
    assert np.array_equal(perm2, np.arange(n)) and np.array_equal(cs2, cs) and np.array_equal(pos2, pos_s)


def test_lattice_density_is_analytic(pkg, O):
    """Interior particle of the 0.02 lattice, R = 0.04, W(0) excluded (Q1): sum over the 32 lattice
    neighbours within the support of m0 * W -- evaluated here in float64."""
    sc = pkg.scene.make_scene("config0")
    p = sc.params
    g = O.grid(p.cell_size, p.cell_length)
    ps, _, _, cs, _ = O.neighbor_search(sc.fluid, np.zeros_like(sc.fluid), g)
    pb, _, _, csb, _ = O.neighbor_search(sc.boundary, None, g)
    A = O.SceneArrays(ps, np.full(ps.shape[0], p.m0, np.float32), cs, pb, np.zeros(pb.shape[0], np.float32), csb, g, p.radius)
    dens = O.density(A)
    R, s = float(p.radius), 0.02
    acc = 0.0
    for i in range(-2, 3):
        for j in range(-2, 3):
            for k in range(-2, 3):
                r = s * (i * i + j * j + k * k) ** 0.5
                q = 2 * r / R
                if r == 0 or q > 2:
                    continue
                a = 0.25 / (np.pi * R ** 3)
                acc += p.m0 * a * ((2 - q) ** 3 if q > 1 else ((3 * q - 6) * q * q + 4))
    interior = float(np.median(dens[dens > 0.99 * dens.max()]))   # float32 lattice coordinates carry ~1e-6 relative jitter
    assert abs(interior - acc) <= 1e-5 * acc


def test_pressure_force_conserves_momentum_and_pbd_rest_state(pkg, O):
    sc = pkg.scene.make_scene("mini", jitter=0.004)
    p = sc.params
    g = O.grid(p.cell_size, p.cell_length)
    ps, _, _, cs, _ = O.neighbor_search(sc.fluid, np.zeros_like(sc.fluid), g)
    # empty boundary range: fluid-fluid forces are antisymmetric -> total momentum change vanishes
    csb = np.zeros_like(cs)
    A = O.SceneArrays(ps, np.full(ps.shape[0], p.m0, np.float32), cs, np.zeros((1, 3), np.float32), np.zeros(1, np.float32), csb, g, p.radius)
    dens = O.density(A) * np.float32(1.3)
    pres = O.pressure(dens, p.rho0, 0.5)     # soft enough that no particle hits the MAX_A clamp
    v = O.pressure_force(A, dens, pres, np.zeros_like(ps), p.dt)
    assert np.abs(v).max() > 0 and np.linalg.norm(v, axis=1).max() / p.dt < 1000.0
    assert np.abs(v.astype(np.float64).sum(0)).max() <= 1e-4 * np.abs(v).astype(np.float64).sum()
    d, lam = O.pbd_density_lambda(A, p.rho0, 0.75)
    assert np.all(lam[d <= p.rho0] == 0.0)


@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
def test_oracle_pinned_to_reference_cuda_golden(pkg, O, solver):
    """Pins the restatement: mini dam-break, state after the constructor and after 2 steps, against the
    outputs of the reference's own kernels on an H100 (bit-exact keys; <= 1e-5 on pos / density)."""
    path = os.path.join(GOLDEN, f"mini_{solver}.npz")
    if not os.path.exists(path):
        pytest.skip("golden fixture not generated yet")
    gold = np.load(path)
    sc = pkg.scene.benchmark_scene("mini", solver)
    s = O.OracleSystem(sc, hash_rcp=_rcp_from_meta())
    for k in range(int(gold["steps"]) + 1):
        assert np.array_equal(s.field("p2c"), gold[f"p2c_{k}"]), f"step {k}"
        assert_close(s.field("pos"), gold[f"pos_{k}"], what=f"{solver} step {k} pos")
        assert_close(s.field("density"), gold[f"density_{k}"], what=f"{solver} step {k} density")
        assert relerr(s.field("vel"), gold[f"vel_{k}"]) <= 1e-3 or np.abs(gold[f"vel_{k}"]).max() == 0
        s.step()
    assert_close(s.field("massB"), gold["massB"], what="boundary mass")
    assert np.array_equal(s.field("p2cB"), gold["p2cB"])
    s.close()


def oracle_per_element_ratios(O, A, p, rng):
    """Every oracle sweep operator on A against the float64 reference (tests/ref64.py), per element.  Returns the
    largest |x - ref| / mag of each output."""
    import ref64
    P = ref64.Pairs(A)
    n = A.n
    F = np.float32
    vel = (0.5 * np.sin(7.0 * A.posF) + 0.05 * rng.standard_normal((n, 3))).astype(F)
    out = {}

    def dv(x, base):
        return np.asarray(x, np.float64) - np.asarray(base, np.float64), ref64.f32_spacing(x)

    dens = O.density(A)
    out["density"] = ref64.ratio(dens, ref64.density(P))
    dhi = (dens * F(1.3)).astype(F)
    pres = O.pressure(dhi, p.rho0, p.stiff)
    x, fl = dv(O.pressure_force(A, dhi, pres, vel, p.dt), vel)
    out["pressure force"] = ref64.ratio(x, ref64.pressure_force_dv(P, dhi, pres, p.dt), fl)
    out["viscosity"] = ref64.ratio(O.viscosity(A, vel, p.rho0, p.visc, p.dt), ref64.viscosity_dv(P, vel, p.rho0, p.visc, p.dt))
    cg = O.color_grad(A, p.rho0, p.rho_boundary)
    out["colour gradient"] = ref64.ratio(cg, ref64.color_grad(P, p.rho0, p.rho_boundary))
    x, fl = dv(O.surface(A, cg, np.zeros_like(vel), p.dt, p.rho0, p.surface_tension, p.air_pressure), 0.0)
    out["surface"] = ref64.ratio(x, ref64.surface_dv(P, cg, p.rho0, p.surface_tension, p.air_pressure, p.dt), fl)
    d, a = O.dfsph_density_alpha(A)
    rd, ra = ref64.dfsph_density_alpha(P)
    out["dfsph density"], out["alpha"] = ref64.ratio(d, rd), ref64.ratio(a, ra)
    e, k = O.dfsph_error(A, vel, d, a, p.dt, p.rho0, "div")
    re_, rk = ref64.dfsph_div_error(P, vel, d, a, p.dt, p.rho0, tau=ref64.TAU)
    out["divergence error"], out["divergence stiffness"] = ref64.ratio(e, re_), ref64.ratio(k, rk)
    x, fl = dv(O.dfsph_correct(A, k, vel, 0.0), vel)
    out["divergence correct"] = ref64.ratio(x, ref64.dfsph_correct_dv(P, k), fl)
    dhi = (d * F(1.28)).astype(F)
    e, k = O.dfsph_error(A, vel, dhi, a, p.dt, p.rho0, "den")
    re_, rk = ref64.dfsph_den_error(P, vel, dhi, a, p.dt, p.rho0)
    out["density error"], out["density stiffness"] = ref64.ratio(e, re_), ref64.ratio(k, rk)
    x, fl = dv(O.dfsph_correct(A, k, vel, p.dt), vel)
    out["density correct"] = ref64.ratio(x, ref64.dfsph_correct_dv(P, k, p.dt), fl)
    rho0 = float(np.median(d))         # (PBD: about half the particles above rest density, lambda != 0)
    d, lam = O.pbd_density_lambda(A, rho0, 0.75)
    rd, rl = ref64.pbd_density_lambda(P, rho0, 0.75)
    assert (lam != 0).sum() > n // 4
    out["pbd density"], out["lambda"] = ref64.ratio(d, rd), ref64.ratio(lam, rl)
    out["delta pos"] = ref64.ratio(O.pbd_delta_pos(A, lam, rho0), ref64.pbd_delta_pos(P, lam, rho0))
    x, fl = dv(O.pbd_xsph(A, vel, 0.05, rho0), vel)
    out["xsph"] = ref64.ratio(x, ref64.pbd_xsph_dv(P, vel, 0.05, rho0), fl)
    return out


@pytest.mark.parametrize("masses", ["uniform", "nonuniform"])
@pytest.mark.parametrize("name,jitter", [("mini", 0.004), ("config0", 0.002), ("walls", None)])
def test_oracle_per_element_vs_float64(pkg, O, name, jitter, masses):
    """Every oracle operator against the float64 reference per element (not scale-relative): a wrong term on a
    low-magnitude (surface, boundary-adjacent) particle cannot hide under the bulk's scale.  Jittered scenes (the
    lattice puts pairs exactly at the surface-tension kernel's jump 2r = R); non-uniform masses m0 * U(0.5, 2); "walls":
    a block against all six walls (boundary terms) with particles outside the grid (tests/sweep_driver.py)."""
    from sweep_driver import walls_scene
    sc = walls_scene(pkg) if name == "walls" else pkg.scene.make_scene(name, jitter=jitter)
    p = sc.params
    g = O.grid(p.cell_size, p.cell_length)
    ps, _, _, cs, _ = O.neighbor_search(sc.fluid, np.zeros_like(sc.fluid), g)
    pb, _, _, csb, _ = O.neighbor_search(sc.boundary, None, g)
    mb = O.boundary_mass(pb, csb, g, p.rho_boundary, p.radius)
    rng = np.random.default_rng(5)
    m = np.full(ps.shape[0], p.m0, np.float32)
    if masses == "nonuniform":
        m = (m * rng.uniform(0.5, 2.0, m.shape)).astype(np.float32)
    A = O.SceneArrays(ps, m, cs, pb, mb, csb, g, p.radius)
    ratios = oracle_per_element_ratios(O, A, p, rng)
    print({k: f"{v:.2e}" for k, v in ratios.items()})
    import ref64
    bad = {k: v for k, v in ratios.items() if not v <= ref64.TAU}
    assert not bad, f"outside |x - ref| <= {ref64.TAU:.0e} * mag: {bad}"


def test_oracle_dfsph_iteration_control(pkg, O):
    """Q11: negative thresholds force exactly maxIter iterations; default thresholds stop early or at 20."""
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    s = O.OracleSystem(sc)
    from oracle.oracle import lib
    import ctypes as C
    assert lib().oracle_system_iters(s.h, 0) == 4 and lib().oracle_system_iters(s.h, 1) == 4
    s.close()
    s = O.OracleSystem(pkg.scene.make_scene("mini", solver="dfsph", dt=0.004))
    assert 1 <= lib().oracle_system_iters(s.h, 0) <= 20 and 2 <= lib().oracle_system_iters(s.h, 1) <= 20
    s.close()
