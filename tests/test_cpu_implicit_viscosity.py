"""The float64 reference of the implicit viscosity solve (tests/implicit_visc_ref.py) against closed forms: symmetry and
spectrum of the operator, rigid motion, momentum and energy, a shear mode on a periodic lattice, the explicit stability limit
the GPU tests use, and the exported symbols.  numpy + scipy only."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
from scipy.spatial import cKDTree

import implicit_visc_ref as IV
import ref64
from util import ROOT

R, SPACING, M0, RHO0, RHOB, DT = 0.04, 0.02, 76.596750762082e-6, 1.0, 1.4, 0.004


def _pairs(pos, posB=None, mass=None, massB=None):
    n = pos.shape[0]
    posB = np.zeros((0, 3)) if posB is None else posB
    mass = np.full(n, M0) if mass is None else mass
    massB = np.full(posB.shape[0], 2 * M0) if massB is None else massB
    A = SimpleNamespace(posF=pos, massF=mass, csF=np.array([0, n]), posB=posB, massB=massB, csB=np.array([0, posB.shape[0]]),
                        g=SimpleNamespace(ncells=1), R=R)
    return ref64.Pairs(A), mass


def _block(k=8, jitter=0.004, seed=1):
    g = np.arange(k) * SPACING + 0.1
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    return pos + np.random.default_rng(seed).uniform(-jitter, jitter, pos.shape)


def _wall(k=8):
    g = np.arange(-2, k + 2) * SPACING + 0.1
    x, z = np.meshgrid(g, g, indexing="ij")
    return np.stack([x.ravel(), np.full(x.size, 0.1 - SPACING), z.ravel()], 1)


def _scene(wall, seed=1):
    pos = _block(seed=seed)
    mass = M0 * np.random.default_rng(seed + 10).uniform(0.5, 2.0, pos.shape[0])
    P, m = _pairs(pos, _wall() if wall else None, mass)
    return P, m, pos


@pytest.mark.parametrize("wall", [False, True])
def test_operator_is_mass_self_adjoint_with_eigenvalues_at_least_one(wall):
    """m_i c_ij = m_j c_ji: M A is symmetric (non-uniform masses), and its spectrum in the M inner product is >= 1"""
    P, m, _ = _scene(wall)
    A, _ = IV.assemble(P, 0.05, 0.05, DT, RHO0, RHOB)
    MA = (A.T.multiply(np.repeat(m, 3))).T.tocsr()
    asym = abs(MA - MA.T).max()
    assert asym <= 1e-12 * abs(MA).max()
    lo = IV.spectrum(A, m, "SA")
    assert lo >= 1.0 - 1e-12, lo
    assert IV.spectrum(A, m, "LA") > 1.5          # the scene is viscous enough to matter


def test_rigid_motion_clear_of_walls_is_a_fixed_point():
    """v = V + W x x: d . (v_i - v_j) = d . (W x d) = 0 for every pair, so A v = v and the solve returns v*"""
    P, m, pos = _scene(False)
    A, _ = IV.assemble(P, 0.2, 0.0, DT, RHO0, RHOB)
    v = np.array([0.3, -0.2, 0.1]) + np.cross(np.array([0.5, -1.2, 0.8]), pos)
    assert np.abs((A @ v.ravel()).reshape(-1, 3) - v).max() <= 1e-12 * np.abs(v).max()
    assert np.abs(IV.solve(A, v) - v).max() <= 1e-12 * np.abs(v).max()


@pytest.mark.parametrize("wall", [False, True])
def test_exact_solution_conserves_momentum_and_does_not_gain_energy(wall):
    """nu_b = 0: pair forces are central and antisymmetric, so sum m v and sum m x x v are those of v*; KE does not grow
    (static walls, nu_b > 0 included for the energy)"""
    P, m, pos = _scene(wall, seed=4)
    v0 = np.random.default_rng(5).standard_normal(pos.shape)
    A, _ = IV.assemble(P, 0.1, 0.0, DT, RHO0, RHOB)
    v = IV.solve(A, v0)
    assert np.abs(v - v0).max() > 1e-3                        # the solve does something
    p0, p1 = (m[:, None] * v0).sum(0), (m[:, None] * v).sum(0)
    L0, L1 = (m[:, None] * np.cross(pos, v0)).sum(0), (m[:, None] * np.cross(pos, v)).sum(0)
    scale_p = (m[:, None] * np.abs(v0)).sum()
    scale_L = (m[:, None] * np.abs(np.cross(pos, v0))).sum()
    assert np.abs(p1 - p0).max() <= 1e-12 * scale_p
    assert np.abs(L1 - L0).max() <= 1e-12 * scale_L
    for nub in (0.0, 0.1):
        A, _ = IV.assemble(P, 0.1, nub, DT, RHO0, RHOB)
        v = IV.solve(A, v0)
        assert (m[:, None] * v * v).sum() <= (m[:, None] * v0 * v0).sum() * (1 + 1e-12)


def test_boundary_terms_move_the_fluid_with_a_moving_wall():
    """b_i = v*_i + dt sum_b c_ib d (d . v_b): a wall moving at u drags the fluid at rest towards u, and nothing moves
    with nu_b = 0"""
    P, m, pos = _scene(True)
    vb = np.tile([0.0, 0.3, 0.0], (_wall().shape[0], 1))
    D, _, b, _ = IV.setup(P, np.zeros_like(pos), vb, 0.1, 0.1, DT, RHO0, RHOB)
    A, D2 = IV.assemble(P, 0.1, 0.1, DT, RHO0, RHOB)
    assert np.abs(D - D2).max() <= 1e-12 * np.abs(D).max()
    v = IV.solve(A, b)
    near = np.bincount(P.iB, minlength=P.n) > 0
    mv = (m[:, None] * v).sum(0)
    assert near.any() and np.all(v[near, 1] > 0) and mv[1] > 10 * np.abs(mv[[0, 2]]).max()
    _, _, b0, _ = IV.setup(P, np.zeros_like(pos), vb, 0.1, 0.0, DT, RHO0, RHOB)
    assert np.all(b0 == 0.0)


def test_pcg_matches_the_exact_solution_and_block_jacobi_beats_the_diagonal():
    P, m, pos = _scene(True, seed=7)
    A, D = IV.assemble(P, 0.3, 0.3, DT, RHO0, RHOB)
    v0 = np.random.default_rng(8).standard_normal(pos.shape)
    exact = IV.solve(A, v0)
    x, it, res = IV.pcg(A, D, v0, v0, m, 1e-10, 500)
    assert res <= 1e-10 and it > 2
    assert IV.m_norm(x - exact, m) <= 1e-8 * IV.m_norm(exact, m)
    _, it_d, _ = IV.pcg(A, D, v0, v0, m, 1e-10, 500, precond="diag")
    assert it_d > it
    # a fluid at rest: no iteration, nothing changes
    z = np.zeros_like(v0)
    x, it, res = IV.pcg(A, D, z, z, m, 1e-4, 50)
    assert it == 0 and np.all(x == 0) and res == 0.0


# ---- a shear mode on a periodic lattice ------------------------------------------------------------------------------------
def _periodic(nx, ny, nz):
    g = lambda k: np.arange(k) * SPACING  # noqa: E731
    pos = np.stack(np.meshgrid(g(nx), g(ny), g(nz), indexing="ij"), -1).reshape(-1, 3)
    box = np.array([nx, ny, nz]) * SPACING
    t = cKDTree(pos, boxsize=box)
    mm = t.sparse_distance_matrix(t, R * (1 + 1e-6), output_type="ndarray")
    i, j = mm["i"].astype(np.int64), mm["j"].astype(np.int64)
    keep = i != j
    i, j = i[keep], j[keep]
    d = pos[i] - pos[j]
    d -= box * np.round(d / box)
    z = np.zeros(0, np.int64)
    P = SimpleNamespace(n=pos.shape[0], R=R, iF=i, jF=j, dF=d, rF=np.sqrt((d ** 2).sum(1)), mF=np.full(i.shape[0], M0),
                        iB=z, jB=z, dB=np.zeros((0, 3)), rB=np.zeros(0), mB=np.zeros(0))
    return P, pos, box


# nu_eff / nu of the discrete operator for v_x = sin(k y) on the lattice of the reference's scenes (spacing 0.02, R = 0.04,
# V = m0 / rho0): the long-wave limit is about 0.83 (the reference's kernel and m0 / rho0 are not normalised to the lattice)
SHEAR_RATIO = {8: 0.79344, 16: 0.82484, 32: 0.83284}


@pytest.mark.parametrize("ny", sorted(SHEAR_RATIO))
def test_shear_mode_decays_like_the_continuum_with_the_recorded_effective_viscosity(ny):
    """The exact solve maps the lattice mode to itself (x only, uniform factor); its factor is 1 / (1 + nu_eff k^2 dt) with
    nu_eff / nu as recorded (DESIGN.md section 2.5), against the continuum's 1 / (1 + nu k^2 dt)"""
    P, pos, box = _periodic(4, ny, 4)
    nu = 1e-3
    k = 2 * np.pi / box[1]
    A, _ = IV.assemble(P, nu, 0.0, DT, RHO0, RHOB)
    v = np.zeros_like(pos)
    v[:, 0] = np.sin(k * pos[:, 1])
    x = IV.solve(A, v)
    fac = float(x[:, 0] @ v[:, 0] / (v[:, 0] @ v[:, 0]))
    assert np.abs(x[:, 1:]).max() <= 1e-12 and np.abs(x[:, 0] - fac * v[:, 0]).max() <= 1e-12
    ratio = (1.0 / fac - 1.0) / (DT * nu * k * k)
    assert abs(ratio - SHEAR_RATIO[ny]) <= 1e-4, ratio
    assert fac > 1.0 / (1.0 + nu * k * k * DT)            # decays less than the continuum: nu_eff < nu


# ---- the explicit limit on the reference scene -----------------------------------------------------------------------------
# 2 / (dt lambda_max) of the same operator (nu = nu_b = 1 per unit nu) on the "mini" DFSPH dam break at dt = 0.004: an explicit
# Euler step of the same term is unstable above this nu.  tests/test_gpu_implicit_viscosity.py runs the implicit solve at >= 10x.
NU_CRIT_MINI = 0.011992


def test_explicit_stability_limit_of_the_mini_scene(pkg):
    sc = pkg.scene.make_scene("mini", solver="dfsph")
    p = sc.params
    bpos = sc.boundary.astype(np.float64)
    t = cKDTree(bpos)
    mm = t.sparse_distance_matrix(t, p.radius * (1 + 1e-6), output_type="ndarray")
    w, _ = ref64.W(np.sqrt(((bpos[mm["i"]] - bpos[mm["j"]]) ** 2).sum(1)), p.radius)
    mB = p.rho_boundary / np.maximum(ref64.EPS, np.bincount(mm["i"], w, bpos.shape[0]))      # SPHSystem.cu:79-105
    m = np.full(sc.fluid.shape[0], p.m0)
    P, _ = _pairs(sc.fluid.astype(np.float64), bpos, m, mB)
    P.R = p.radius
    A, _ = IV.assemble(P, 1.0, 1.0, 1.0, p.rho0, p.rho_boundary)
    lam = IV.spectrum(A, m, "LA") - 1.0
    nu_crit = 2.0 / (float(np.float32(p.dt)) * lam)
    assert abs(nu_crit - NU_CRIT_MINI) <= 1e-4 * NU_CRIT_MINI, nu_crit


# ---- exported symbols --------------------------------------------------------------------------------------------------------
def test_exported_symbols(built):
    from cpp_fluid_particles_b200 import capi
    L = C.CDLL(capi.LIBSPHK)
    for name in ("sphk_implicit_viscosity_work_floats", "sphk_implicit_viscosity", "sphk_implicit_viscosity_stats",
                 "sphk_visc_implicit_setup", "sphk_visc_implicit_matvec"):
        assert hasattr(L, name), name
        assert name in capi.SPHK_FUNCTIONS
    H = C.CDLL(capi.LIBHOST, mode=C.RTLD_LOCAL)
    for name in ("sph_app_set_implicit_viscosity", "sph_app_viscosity_stats"):
        assert hasattr(H, name), name
        assert name in capi.SPH_APP_FUNCTIONS
    L.sphk_implicit_viscosity_work_floats.restype = C.c_longlong
    assert L.sphk_implicit_viscosity_work_floats(C.c_int(1000)) == 64 + 6 * 1024 + 21 * 1000
    assert L.sphk_implicit_viscosity_work_floats(C.c_int(-1)) < 0
    for h in ("sphk.h", "sph_app.h"):
        assert os.path.exists(os.path.join(ROOT, "include", h))


# ---- the layers that refuse the setting ----------------------------------------------------------------------------------------
def test_slab_system_refuses_implicit_viscosity(pkg):
    from cpp_fluid_particles_b200 import slabs
    obj = object.__new__(slabs.SlabSystem)
    obj.implicit_nu = 0.0
    with pytest.raises(ValueError):
        obj.implicit_nu = 0.1
    assert obj.implicit_nu == 0.0


@pytest.mark.parametrize("extra", [["-1"], ["nan"], ["0.1", "--ranks", "2"], ["0.1", "--float", "0.5"]])
def test_headless_refuses_bad_settings(built, extra):
    """refused while parsing, before any CUDA call: negative or NaN NU, --ranks (slab ranks), --float (dynamic body)"""
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    r = subprocess.run([cli, "--frames", "0", "--implicit-viscosity"] + extra, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=60)
    assert r.returncode == 2, r.stderr
