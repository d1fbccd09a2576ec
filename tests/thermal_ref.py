"""A float64 reference of heat transfer (DESIGN.md section 2.10) -- TEST INFRASTRUCTURE ONLY (numpy + scipy).

From the explicit pair lists of ref64.Pairs, with d = x_i - x_j, r = |d|, f the kernel gradient factor (grad W = d f, f <= 0) and
eta^2 = 0.0025 R^2:
    dT_i/dt = sum_j c_ij (T_j - T_i),   c_ij = -2 alpha V_j f r^2 / (r^2 + eta^2)
    fluid j: V_j = m_j / rho0;  boundary j of group g: V_b = m_b / rho_B, alpha -> h_g alpha, T_j -> T_g
Every value comes with the magnitude its float32 rounding scales with (the ref64 convention), for per-element bounds.
"""
from __future__ import annotations

import math

import numpy as np

EPS = 1e-6
COP = 100.0                     # SPHK_HEAT_COP


def grad_factor(r, R):
    """f with grad W = d f (the repository's cubic kernel, ref64.grad_W's scalar)"""
    q = 2.0 * np.asarray(r, np.float64) / R
    p = np.where(q > 1.0, (12.0 - 3.0 * q) * q - 12.0, (9.0 * q - 12.0) * q)
    return np.where(q > 2.0, 0.0, p / (np.pi * (q + EPS) * R ** 5))


def coefficients(P, alpha, rho0, rhoB, gB=None, groups=((0.0, 0.0),)):
    """(c_ij of the fluid pairs, c_ib of the boundary pairs, T_g of the boundary pairs)"""
    R = P.R
    eta2 = 0.0025 * R * R
    cF = -2.0 * alpha * (P.mF / rho0) * grad_factor(P.rF, R) * P.rF ** 2 / (P.rF ** 2 + eta2)
    g = np.zeros(P.jB.shape[0], np.int64) if gB is None else np.asarray(gB, np.int64)[P.jB]
    tab = np.asarray(groups, np.float64).reshape(-1, 2)
    if g.size and g.max() >= tab.shape[0]:          # groups past the table are adiabatic
        tab = np.concatenate([tab, np.zeros((g.max() + 1 - tab.shape[0], 2))])
    tg, hg = tab[g, 0], tab[g, 1]
    cB = -2.0 * alpha * hg * (P.mB / rhoB) * grad_factor(P.rB, R) * P.rB ** 2 / (P.rB ** 2 + eta2)
    return cF, cB, tg


def conduction(P, T, alpha, rho0, rhoB, gB=None, groups=((0.0, 0.0),)):
    """dict(value, mag, csum): dT/dt per particle, its rounding magnitude and sum_j c_ij"""
    T = np.asarray(T, np.float64)
    cF, cB, tg = coefficients(P, alpha, rho0, rhoB, gB, groups)
    n = P.n
    dF, dB = T[P.jF] - T[P.iF], tg - T[P.iB]
    value = np.bincount(P.iF, cF * dF, n) + np.bincount(P.iB, cB * dB, n)
    mag = (np.bincount(P.iF, np.abs(cF) * (np.abs(T[P.jF]) + np.abs(T[P.iF])), n)
           + np.bincount(P.iB, np.abs(cB) * (np.abs(tg) + np.abs(T[P.iB])), n))
    csum = np.bincount(P.iF, cF, n) + np.bincount(P.iB, cB, n)
    return {"value": value, "mag": mag, "csum": csum}


def substeps(alpha, h_max, R, dt):
    """sphk_heat_substeps: max(1, ceil(dt COP alpha (1 + h_max) / R^2))"""
    return max(1, int(math.ceil(dt * COP * alpha * (1.0 + h_max) / (R * R))))


def run(P, T, alpha, rho0, rhoB, dt, steps, gB=None, groups=((0.0, 0.0),), h_max=None):
    """the explicit Jacobi substeps of `steps` steps of length dt on fixed positions"""
    T = np.asarray(T, np.float64).copy()
    hm = max([h for _, h in groups]) if h_max is None else h_max
    k = substeps(alpha, hm, P.R, dt)
    for _ in range(steps * k):
        T = T + (dt / k) * conduction(P, T, alpha, rho0, rhoB, gB, groups)["value"]
    return T


def nu_of_t(T, nu_ref, e, t_ref, nu_min, nu_max):
    """clamp(nu_ref exp(-e (T - t_ref)), nu_min, nu_max) in float64 (a NaN lands on nu_max)"""
    with np.errstate(over="ignore", invalid="ignore"):
        raw = nu_ref * np.exp(-e * (np.asarray(T, np.float64) - t_ref))
    return np.where(~(raw < nu_max), nu_max, np.maximum(raw, nu_min))
