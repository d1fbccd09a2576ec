"""A float64 reference of the non-Newtonian viscosity solve (DESIGN.md section 2.9) -- TEST INFRASTRUCTURE ONLY (numpy + scipy).

Extends implicit_visc_ref (the constant-nu solve) with what the per-particle viscosity adds, from the explicit pair lists of
ref64.Pairs:
    shear rate   G_i = sum_j V_j (v_j - v_i) (x) gradW_ij,  M_i = -sum_j V_j g d d^T   (boundary pairs only when beta > 0)
                 grad v_i = G_i M_i^-1, or G_i 3 / tr M_i where det M_i < THETA (tr M_i / 3)^3
                 gamma_dot_i = sqrt(2 E:E),  E = (grad v + grad v^T) / 2
    models       Cross and Herschel-Bulkley (Papanastasiou), clamped to [nu_min, nu_max]
    pairs        fluid nu_ij = (nu_i + nu_j) / 2, boundary beta nu_i
Every value comes with the magnitude its float32 rounding scales with (the ref64 convention), for per-element bounds.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps

import implicit_visc_ref as IV

THETA = 0.01                    # SPHK_RHEO_THETA
CROSS, HB = 1, 2                # SPHK_RHEOLOGY_*


# ---- models ------------------------------------------------------------------------------------------------------------------
def model_nu(model, params, nu_min, nu_max, g):
    """(nu, at the nu_max clamp) of the model in float64 for the shear rates g (any shape); a NaN rate lands on nu_max"""
    g = np.asarray(g, np.float64)
    p = [float(x) for x in params]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if model == CROSS:
            nu0, nu_inf, lam, m = p[:4]
            raw = nu_inf + (nu0 - nu_inf) / (1.0 + np.power(lam * g, m))
        elif model == HB:
            K, n, tau, mr = p[:4]
            power = K * np.power(g, n - 1.0) if K > 0 else np.zeros_like(g)
            yield_ = np.where(g > 0, tau * (-np.expm1(-mr * g) / np.where(g > 0, g, 1.0)), tau * mr)
            raw = power + yield_
        else:
            raise ValueError(model)
    at_max = ~(raw < nu_max)
    return np.where(at_max, float(nu_max), np.maximum(raw, nu_min)), at_max


# ---- shear rate --------------------------------------------------------------------------------------------------------------
def _outer_sum_full(n, i, u, w):
    """sum over the pairs of each particle of u (x) w, as (n, 3, 3)"""
    out = np.zeros((n, 3, 3))
    for a in range(3):
        for b in range(3):
            out[:, a, b] = np.bincount(i, u[:, a] * w[:, b], n)
    return out


def shear(P, vel, vel_b, beta, rho0, rho_b):
    """dict of the shear sweep: grad (n, 3, 3) with its magnitude, gamma with its magnitude, flag (1 = scalar normalisation),
    near (det M within rounding of the switch: both branches acceptable) and the other branch's grad / gamma there"""
    v = np.asarray(vel, np.float64)
    vb = np.asarray(vel_b, np.float64)
    g, gs = IV.grad_factor(P.rF, P.R)
    VF = P.mF / rho0
    u = v[P.jF] - v[P.iF]
    um = np.abs(v[P.jF]) + np.abs(v[P.iF])
    w, wm = (VF * g)[:, None] * P.dF, (VF * gs)[:, None] * np.abs(P.dF)
    G = _outer_sum_full(P.n, P.iF, u, w)
    Gm = _outer_sum_full(P.n, P.iF, um, wm)
    M = -_outer_sum_full(P.n, P.iF, w, P.dF)
    Mm = _outer_sum_full(P.n, P.iF, wm, np.abs(P.dF))
    if beta > 0 and P.iB.size:
        gb, gbs = IV.grad_factor(P.rB, P.R)
        VB = P.mB / rho_b
        ub = vb[P.jB] - v[P.iB]
        ubm = np.abs(vb[P.jB]) + np.abs(v[P.iB])
        wb, wbm = (VB * gb)[:, None] * P.dB, (VB * gbs)[:, None] * np.abs(P.dB)
        G += _outer_sum_full(P.n, P.iB, ub, wb)
        Gm += _outer_sum_full(P.n, P.iB, ubm, wbm)
        M -= _outer_sum_full(P.n, P.iB, wb, P.dB)
        Mm += _outer_sum_full(P.n, P.iB, wbm, np.abs(P.dB))
    tr = np.trace(M, axis1=1, axis2=2)
    det = np.linalg.det(M)
    t3 = (tr / 3.0) ** 3
    corrected = (tr > 0) & (det >= THETA * t3)
    # rounding of det relative to (tr/3)^3: |d det| <= sum |cofactor| |dM|, dM ~ 2e-6 Mm (generous: the branch is accepted both ways)
    cof = np.abs(np.linalg.inv(np.where((np.abs(det) > 0)[:, None, None], M, np.eye(3)[None])) * det[:, None, None])
    ddet = 1e-5 * (cof * Mm).sum((1, 2)) + 3.0 * THETA * (tr / 3.0) ** 2 * 1e-5 * np.trace(Mm, axis1=1, axis2=2) / 3.0
    near = (tr > 0) & (np.abs(det - THETA * t3) <= ddet)

    def branch(corr):
        Minv = np.zeros_like(M)
        ok = corr & (np.abs(det) > 0)
        Minv[ok] = np.linalg.inv(M[ok])
        sc = np.where(tr > 0, 3.0 / np.where(tr > 0, tr, 1.0), 0.0)
        Minv[~corr] = np.eye(3)[None] * sc[~corr, None, None]
        L = G @ Minv
        Lm = Gm @ np.abs(Minv) + np.abs(L) @ Mm @ np.abs(Minv)
        E = 0.5 * (L + np.transpose(L, (0, 2, 1)))
        gam = np.sqrt(2.0 * (E * E).sum((1, 2)))
        gm = np.sqrt(2.0) * np.sqrt((Lm * Lm).sum((1, 2)))
        return L, Lm, gam, gm

    L, Lm, gam, gm = branch(corrected)
    La, Lam, gama, gma = branch(~corrected)
    return dict(grad=L, grad_mag=Lm, gamma=gam, gamma_mag=gm, flag=(~corrected).astype(np.int32), near=near,
                grad_alt=np.where(near[:, None, None], La, L), grad_alt_mag=np.where(near[:, None, None], Lam, Lm),
                gamma_alt=np.where(near, gama, gam), gamma_alt_mag=np.where(near, gma, gm), det=det, tr=tr)


# ---- the pair coefficients with a per-particle nu ----------------------------------------------------------------------------
def coefficients(P, nu, beta, rho0, rho_b, mean=True):
    """(c, size of c) of the fluid pairs (nu_ij = (nu_i + nu_j) / 2, or nu_j with mean=False) and of the boundary pairs
    (beta nu_i)"""
    nu = np.asarray(nu, np.float64)
    den = lambda r: r * r + 0.01 * P.R * P.R  # noqa: E731
    g, gs = IV.grad_factor(P.rF, P.R)
    gb, gbs = IV.grad_factor(P.rB, P.R)
    nij = 0.5 * (nu[P.iF] + nu[P.jF]) if mean else nu[P.jF]
    vF = nij * P.mF / rho0
    vB = beta * nu[P.iB] * P.mB / rho_b
    return (-10.0 * vF * g / den(P.rF), 10.0 * vF * gs / den(P.rF)), (-10.0 * vB * gb / den(P.rB), 10.0 * vB * gbs / den(P.rB))


def setup(P, vel, vel_b, nu, beta, dt, rho0, rho_b):
    """(D (n, 3, 3), mag of D, b, mag of b) of OpViscImplicitSetupField"""
    (cF, sF), (cB, sB) = coefficients(P, nu, beta, rho0, rho_b)
    S = IV._outer_sum(P, P.iF, P.dF, cF) + IV._outer_sum(P, P.iB, P.dB, cB)
    mS = IV._outer_sum(P, P.iF, np.abs(P.dF), sF) + IV._outer_sum(P, P.iB, np.abs(P.dB), sB)
    D = np.eye(3)[None] + dt * S
    vb = np.asarray(vel_b, np.float64)[P.jB]
    dvb = (P.dB * vb).sum(1)
    sdvb = (np.abs(P.dB) * np.abs(vb)).sum(1)
    bt = np.stack([np.bincount(P.iB, cB * dvb * P.dB[:, k], P.n) for k in range(3)], 1)
    bm = np.stack([np.bincount(P.iB, sB * sdvb * np.abs(P.dB[:, k]), P.n) for k in range(3)], 1)
    return D, dt * mS, np.asarray(vel, np.float64) + dt * bt, dt * bm


def matvec(P, D, p, nu, dt, rho0):
    """((A p), mag) of OpViscImplicitMatvecField with the given D (n, 3, 3)"""
    (cF, sF), _ = coefficients(P, nu, 0.0, rho0, 1.0)
    p = np.asarray(p, np.float64)
    pj = p[P.jF]
    t = cF * (P.dF * pj).sum(1)
    ts = sF * (np.abs(P.dF) * np.abs(pj)).sum(1)
    off = np.stack([np.bincount(P.iF, t * P.dF[:, k], P.n) for k in range(3)], 1)
    offm = np.stack([np.bincount(P.iF, ts * np.abs(P.dF[:, k]), P.n) for k in range(3)], 1)
    Dp = np.einsum("nab,nb->na", D, p)
    Dpm = np.einsum("nab,nb->na", np.abs(D), np.abs(p))
    return Dp - dt * off, Dpm + dt * offm


def assemble(P, nu, beta, dt, rho0, rho_b, mean=True):
    """A (3n x 3n, CSR) and D (n, 3, 3) with the per-particle nu (mean=False: nu_j instead of the mean, not self-adjoint)"""
    (cF, _), (cB, _) = coefficients(P, nu, beta, rho0, rho_b, mean)
    D = np.eye(3)[None] + dt * (IV._outer_sum(P, P.iF, P.dF, cF) + IV._outer_sum(P, P.iB, P.dB, cB))
    rows, cols, vals = [], [], []
    ii = np.arange(P.n)
    for a in range(3):
        for b in range(3):
            rows += [3 * ii + a, 3 * P.iF + a]
            cols += [3 * ii + b, 3 * P.jF + b]
            vals += [D[:, a, b], -dt * cF * P.dF[:, a] * P.dF[:, b]]
    A = sps.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * P.n, 3 * P.n))
    return A, D


def m_dot(u, w, mass):
    """<u, w>_M in float64"""
    return float((np.repeat(np.asarray(mass, np.float64), 3) * np.ravel(u) * np.ravel(w)).sum())
