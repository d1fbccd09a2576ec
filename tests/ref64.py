"""A float64, per-element reference of every sweep operator -- TEST INFRASTRUCTURE ONLY (numpy + scipy, no GPU).

The CPU oracle (oracle/sph_oracle.c) restates the reference kernels loop for loop in float32, and the parity tests compare
it with the GPU scale-relative (max |a - b| / max |b|).  A wrong term on low-magnitude particles can hide under that scale.
This module evaluates the same operators (the reference lines the oracle cites, with their quirks: W(0) = 0 (Q1), the
boundary terms of each kernel, the SPHK_MAX_A clamp, the divergence-error zeroing of DFSPHSolver.cu:302-303, rho0 passed
through `bool` (Q4), Jacobi XSPH (Q5)) in float64 from explicit pair lists, and returns for every output element its value
and its magnitude  mag = sum_j |term_j|  (propagated through the epilogue of the operator).  A float32 implementation that
forms the same sum in any order is within a few 1e-7 * mag of the value, element by element:

    |x - value| <= tau * mag + floor

Two places are discontinuous and are accepted on either side (`alt`): the jump of the surface-tension kernel at 2r = R
(pairs within 4e-6 R of it) and the zeroing of the divergence error (elements whose test rho + dt e < rho0 lies within
the bound of its threshold).  Every other branch (max(0, .), the acceleration clamp, the PBD rho > rho0 test) is continuous
in the value, and `mag` is defined the same on both sides of it.

Neighbour rule: j counts for i iff j lies in the grid (key(j) < ncells, i.e. its sorted slot is below cell_start[ncells]);
the cell length is 1.01 R, so every in-grid pair within R sits in adjacent cells -- also for an i outside the grid.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.spatial import cKDTree

EPS = 1e-6            # global.h:21
MAX_A = 1000.0        # global.h:26
# the per-element bound of the float32 sweeps (CPU oracle and GPU kernels); largest observed ratios: DESIGN.md section 2
TAU = 2e-6
ST_JUMP = 4e-6        # half-width (in units of R) of the window around 2r = R where both surface-tension branches count


@dataclasses.dataclass
class R64:
    value: np.ndarray
    mag: np.ndarray
    alt: np.ndarray | None = None      # the value on the other side of a discontinuity (NaN-free, == value elsewhere)
    floor: np.ndarray | float = 0.0    # absolute allowance for the float32 rounding of an epilogue that adds O(1) inputs


class Pairs:
    """Fluid-fluid and fluid-boundary pairs within R of the sorted arrays (any object with posF, massF, csF, posB, massB,
    csB, g.ncells, R -- e.g. oracle.SceneArrays)."""

    def __init__(self, A, masses=None):
        self.R = R = float(A.R)
        nc = int(A.g.ncells)
        x = np.asarray(A.posF, np.float64)
        xb = np.asarray(A.posB, np.float64)
        self.n = x.shape[0]
        mF = np.asarray(A.massF if masses is None else masses, np.float64)
        mB = np.asarray(A.massB, np.float64)
        inF, inB = int(A.csF[nc]), int(A.csB[nc])
        cut = R * (1.0 + 1e-6)
        every = cKDTree(x)

        def pairs(y, count):
            if count == 0:
                return np.zeros(0, np.int64), np.zeros(0, np.int64)
            m = every.sparse_distance_matrix(cKDTree(y[:count]), cut, output_type="ndarray")
            return m["i"].astype(np.int64), m["j"].astype(np.int64)

        i, j = pairs(x, inF)
        keep = i != j                  # the self pair contributes exactly 0 to every operator
        self.iF, self.jF = i[keep], j[keep]
        self.iB, self.jB = pairs(xb, inB)
        self.dF = x[self.iF] - x[self.jF]
        self.dB = x[self.iB] - xb[self.jB]
        self.rF = np.sqrt((self.dF ** 2).sum(1))
        self.rB = np.sqrt((self.dB ** 2).sum(1))
        self.mF, self.mB = mF[self.jF], mB[self.jB]

    # sums over the pairs of each particle of (term, size) pairs, scalar or 3-vector: (value, mag = sum of sizes)
    def sum(self, i, t):
        v, s = t
        if v.ndim == 1:
            return np.bincount(i, v, self.n), np.bincount(i, s, self.n)
        return (np.stack([np.bincount(i, v[:, k], self.n) for k in range(3)], 1),
                np.stack([np.bincount(i, s[:, k], self.n) for k in range(3)], 1))

    def sum2(self, tF, tB=None):
        v, m = self.sum(self.iF, tF)
        if tB is not None:
            vb, mb = self.sum(self.iB, tB)
            v, m = v + vb, m + mb
        return v, m


def mul(c, t):
    """coefficient c (per pair) times a (value, size) term"""
    v, s = t
    c = np.asarray(c, np.float64)
    if v.ndim == 2 and c.ndim == 1:
        c = c[:, None]
    return c * v, np.abs(c) * s


def dot(u, t):
    """u . t for a per-pair 3-vector u and a vector (value, size) term"""
    return (u * t[0]).sum(1), (np.abs(u) * t[1]).sum(1)


# ---- smoothing kernels, CUDAFunctions.cuh:23-54,82-98 -------------------------------------------------------------------
# Each returns (value, size): `size` is the magnitude of the float32 operands the value is formed from.  Near the edge of
# the support the polynomials cancel ((12 - 3q) q - 12 = -3 (2 - q)^2, (2 - q)^3 from a rounded q, R - r), so a float32
# kernel value there carries a rounding error of the order of its operands, not of itself; mag counts every term at
# this size.
def W(r, R):
    q = 2.0 * r / R
    t = 2.0 - q
    outer = q > 1.0
    w = np.where(outer, t ** 3, (3.0 * q - 6.0) * q * q + 4.0)
    ws = np.where(outer, np.abs(t) ** 3 + 3.0 * t * t * q, np.abs(3.0 * q - 6.0) * q * q + 4.0)
    off = (q > 2.0) | (q < EPS)
    a = 0.25 / (np.pi * R ** 3)
    return np.where(off, 0.0, a * w), np.where(off, 0.0, a * ws)


def grad_W(d, r, R):
    q = 2.0 * r / R
    outer = q > 1.0
    s = np.where(outer, (12.0 - 3.0 * q) * q - 12.0, (9.0 * q - 12.0) * q)
    ss = np.where(outer, (12.0 + 3.0 * q) * q + 12.0, (9.0 * q + 12.0) * q)
    c = np.where(q > 2.0, 0.0, 1.0 / (np.pi * (q + EPS) * R ** 5))
    return d * (s * c)[:, None], np.abs(d) * (ss * c)[:, None]


def lap_visc(r, R):
    on = r <= R
    c = 45.0 / (np.pi * R ** 6)
    return np.where(on, c * (R - r), 0.0), np.where(on, c * R, 0.0)


def grad_st(d, x, R, inner):
    """surface-tension kernel gradient with the branch chosen by `inner` (2x <= R in the reference)"""
    e = R - x
    e3x3 = e ** 3 * x ** 3
    es = np.abs(e) ** 2 * x ** 3 * (np.abs(e) + 3.0 * x)
    s = np.where(inner, 2.0 * e3x3 - 0.0156 * R ** 6, e3x3)
    ss = np.where(inner, 2.0 * es + 0.0156 * R ** 6, es)
    c = np.where((x > R) | (x < EPS), 0.0, 136.0241 / (np.pi * R ** 9 * np.maximum(x, EPS)))
    return -d * (c * s)[:, None], np.abs(d) * (c * ss)[:, None]


def _f64(a):
    return np.asarray(a, np.float64)


# ---- WCSPH, BasicSPHSolver.cu ---------------------------------------------------------------------------------------------
def density(P):
    """computeDensity_CUDA, :32-72"""
    return R64(*P.sum2(mul(P.mF, W(P.rF, P.R)), mul(P.mB, W(P.rB, P.R))))


def pressure_force_dv(P, dens, pres, dt):
    """pressureForce_CUDA, :113-165: the velocity change a*dt, a clamped to SPHK_MAX_A (:160-161)"""
    dens, pres = _f64(dens), _f64(pres)
    s = pres / np.maximum(EPS, dens * dens)
    a, m = P.sum2(mul(-P.mF * (s[P.iF] + s[P.jF]), grad_W(P.dF, P.rF, P.R)), mul(-P.mB * s[P.iB], grad_W(P.dB, P.rB, P.R)))
    la = np.sqrt((a ** 2).sum(1))
    scale = np.where(la > MAX_A, MAX_A / np.maximum(la, 1e-300), 1.0)[:, None]
    # the clamp is continuous; a / |a| carries the error of a twice
    return R64(a * scale * dt, m * np.where(scale < 1.0, 2.0 * scale, 1.0) * dt)


def viscosity_dv(P, vel, rho0, visc, dt):
    """viscosity_CUDA, :183-209 (fluid neighbours only): deltaV = visc * a * dt"""
    vel = _f64(vel)
    lv, ls = lap_visc(P.rF, P.R)
    dv = vel[P.jF] - vel[P.iF]
    v, m = P.sum2(((P.mF * lv / rho0)[:, None] * dv, (P.mF * ls / rho0)[:, None] * np.abs(dv)))
    return R64(visc * dt * v, visc * dt * m)


def color_grad(P, rho0, rhoB):
    """computeColorGrad_CUDA, :277-318: c = num / max(eps, den)"""
    VF, VB = P.mF / rho0, P.mB / rhoB
    num, mnum = P.sum2(mul(VF, grad_W(P.dF, P.rF, P.R)), mul(VB, grad_W(P.dB, P.rB, P.R)))
    den, mden = P.sum2(mul(VF, W(P.rF, P.R)), mul(VB, W(P.rB, P.R)))
    dd = np.maximum(EPS, den)[:, None]
    c = num / dd
    return R64(c, mnum / dd + np.abs(c) * mden[:, None] / dd)


def surface_dv(P, cg, rho0, kappa, airP, dt):
    """surfaceTensionAndAirPressure_CUDA, :332-370 (fluid neighbours only): a * dt"""
    cg = _f64(cg)
    cii = (cg ** 2).sum(1)
    lci = np.sqrt(cii)
    ratio = lci / np.maximum(EPS, lci)                # "disable inner particles", :349
    mr = P.mF / (rho0 * rho0)
    inner = 2.0 * P.rF <= P.R
    c1 = 0.25 * mr * kappa * (cii[P.iF] + cii[P.jF])
    v1, m1 = P.sum2(mul(c1, grad_st(P.dF, P.rF, P.R, inner)))
    v2, m2 = P.sum2(mul(airP * mr * ratio[P.iF], grad_W(P.dF, P.rF, P.R)))
    out = R64((v1 + v2) * dt, (m1 + m2) * dt)
    near = np.abs(2.0 * P.rF - P.R) <= 2.0 * ST_JUMP * P.R
    if near.any():
        sel = np.flatnonzero(near)
        t = c1[sel][:, None] * grad_st(P.dF[sel], P.rF[sel], P.R, inner[sel])[0]
        to = c1[sel][:, None] * grad_st(P.dF[sel], P.rF[sel], P.R, ~inner[sel])[0]
        delta = np.stack([np.bincount(P.iF[sel], (to - t)[:, k], P.n) for k in range(3)], 1)
        out.alt = out.value + delta * dt
    return out


# ---- DFSPH, DFSPHSolver.cu ------------------------------------------------------------------------------------------------
def _gradient_sums(P, boundary_in_lam):
    gF = mul(P.mF, grad_W(P.dF, P.rF, P.R))
    gB = mul(P.mB, grad_W(P.dB, P.rB, P.R))
    gs, mgs = P.sum2(gF, gB)
    lamF = ((gF[0] ** 2).sum(1), 2.0 * (np.abs(gF[0]) * gF[1]).sum(1))
    lamB = ((gB[0] ** 2).sum(1), 2.0 * (np.abs(gB[0]) * gB[1]).sum(1)) if boundary_in_lam else None
    lam, mlam = P.sum2(lamF, lamB)
    S = (gs ** 2).sum(1) + lam
    mS = 2.0 * (np.abs(gs) * mgs).sum(1) + mlam
    return S, mS


def dfsph_density_alpha(P):
    """computeDensityAlpha_CUDA, :212-249: (density, alpha); the boundary is excluded from the second term (:218)"""
    S, mS = _gradient_sums(P, False)
    Sd = np.maximum(EPS, S)
    return density(P), R64(-1.0 / Sd, mS / (Sd * Sd))


def _divergence(P, vel):
    """the shared sum of :281-300 / :94-110: sum_j m_j (v_i - v_j) . gradW (boundary: v_j = 0)"""
    vel = _f64(vel)
    tF = mul(P.mF, dot(vel[P.iF] - vel[P.jF], grad_W(P.dF, P.rF, P.R)))
    tB = mul(P.mB, dot(vel[P.iB], grad_W(P.dB, P.rB, P.R)))
    return P.sum2(tF, tB)


def dfsph_div_error(P, vel, dens, alpha, dt, rho0, tau):
    """computeDivergenceError_CUDA, :281-306: (error, stiffness).  The zeroing of :302-303 is a jump: elements whose test
    lies within tau * mag (+ the float32 rounding of rho + dt e) of its threshold accept both outcomes."""
    dens, alpha = _f64(dens), _f64(alpha)
    e, m = _divergence(P, vel)
    e = np.maximum(0.0, e)
    below = dens <= rho0
    zero = (dens + dt * e < rho0) & below
    val = np.where(zero, 0.0, e)
    near = below & (np.abs(dens + dt * e - rho0) <= dt * tau * m + 2.0 * float(np.spacing(np.float32(rho0))))
    alt = np.where(near, np.where(zero, e, 0.0), val)
    return R64(val, m, alt), R64(val * alpha, m * np.abs(alpha), alt * alpha)


def dfsph_den_error(P, vel, dens, alpha, dt, rho0):
    """computeDensityError_CUDA, :94-116: e = max(0, dt * div + rho - rho0); (error, stiffness)"""
    dens, alpha = _f64(dens), _f64(alpha)
    s, m = _divergence(P, vel)
    e = np.maximum(0.0, dt * s + dens - rho0)
    me = dt * m
    # rho and rho0 enter as inputs, not as sums: the float32 epilogue adds the rounding of (dt * div + rho) and of the
    # difference, each at most one float32 spacing -- an absolute floor, not a share of tau * mag
    fe = f32_spacing(np.abs(dens) + me) + f32_spacing(e)
    k = e * alpha
    return R64(e, me, floor=fe), R64(k, me * np.abs(alpha), floor=fe * np.abs(alpha) + f32_spacing(k))


def dfsph_correct_dv(P, stiff, dt=None):
    """correctDivergenceError_CUDA (:308-329, dt None: vel += a) / correctDensityError_CUDA (:118-158, vel += a / dt)"""
    k = _f64(stiff)
    a, m = P.sum2(mul(P.mF * (k[P.iF] + k[P.jF]), grad_W(P.dF, P.rF, P.R)), mul(P.mB * k[P.iB], grad_W(P.dB, P.rB, P.R)))
    s = 1.0 if dt is None else 1.0 / dt
    return R64(a * s, m * s)


# ---- PBD, PBDSolver.cu ----------------------------------------------------------------------------------------------------
def pbd_density_lambda(P, rho0, relaxation):
    """computeDensityLambda_CUDA, :127-168 (Q4: the gradient is divided by (bool) rho0 = 1; boundary terms included)"""
    S, mS = _gradient_sums(P, True)
    S = S + EPS
    den = density(P)
    C = den.value / rho0 - 1.0
    l = np.where(den.value > rho0, -C / S, 0.0) * relaxation
    ml = relaxation * (den.mag / rho0 / S + np.abs(C) * mS / (S * S))    # continuous at rho = rho0
    return den, R64(l, ml)


def pbd_delta_pos(P, lam, rho0):
    """computeDeltaPos_CUDA, :170-210: deltaPos = a / rho0"""
    lam = _f64(lam)
    a, m = P.sum2(mul(P.mF * (lam[P.iF] + lam[P.jF]), grad_W(P.dF, P.rF, P.R)), mul(P.mB * lam[P.iB], grad_W(P.dB, P.rB, P.R)))
    return R64(a / rho0, m / rho0)


def pbd_xsph_dv(P, vel, c, rho0):
    """XSPHViscosity_CUDA, :89-115, Jacobi (Q5): v_new - v = c * sum_j m_j (v_j - v_i) W / rho0"""
    vel = _f64(vel)
    w, ws = W(P.rF, P.R)
    dv = vel[P.jF] - vel[P.iF]
    v, m = P.sum2(((P.mF * w)[:, None] * dv, (P.mF * ws)[:, None] * np.abs(dv)))
    return R64(c * v / rho0, c * m / rho0)


# ---- the per-element comparison ---------------------------------------------------------------------------------------------
def ratio(x, ref: R64, floor=0.0):
    """largest |x - value| / mag over the elements (the observed tau); elements that match `alt` better are measured
    against it; the absolute `floor` (e.g. the float32 spacing of a velocity the change was added to) is taken off first."""
    x = np.asarray(x, np.float64)
    d = np.abs(x - ref.value)
    if ref.alt is not None:
        d = np.minimum(d, np.abs(x - ref.alt))
    d = np.maximum(d - floor - ref.floor, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(ref.mag > 0, d / ref.mag, np.where(d > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def assert_per_element(x, ref: R64, tau, what, floor=0.0):
    """|x - value| <= tau * mag + floor for every element (or against alt)"""
    x = np.asarray(x, np.float64)
    lim = tau * ref.mag + floor + ref.floor
    ok = np.abs(x - ref.value) <= lim
    if ref.alt is not None:
        ok |= np.abs(x - ref.alt) <= lim
    if not ok.all():
        bad = np.argwhere(~ok)
        k = tuple(bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} element(s) outside |x - ref| <= {tau:.0e} * mag + floor; first {k}: "
                             f"x = {x[k]:.9g}, ref = {ref.value[k]:.9g}, mag = {ref.mag[k]:.3g} "
                             f"(largest ratio {ratio(x, ref, floor):.3g})")


def f32_spacing(a):
    """the float32 spacing of each element: the rounding floor of a quantity added to a float32 value of this size"""
    return np.spacing(np.abs(np.asarray(a, np.float32))).astype(np.float64)
