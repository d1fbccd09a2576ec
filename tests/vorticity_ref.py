"""Float64 per-element reference of the vorticity-confinement sweeps (sphk_vorticity, sphk_vorticity_confinement) -- TEST
INFRASTRUCTURE ONLY, in the style of ref64.py (explicit pair lists, value and mag = sum_j |term_j| per element).

    omega_i = sum_j V_j (v_i - v_j) x gradW_ij                   V_j = m_j / rho0, fluid neighbours only
    eta_i   = sum_j V_j (|omega_j| - |omega_i|) gradW_ij
    dv_i    = dt * eps * (N_i x omega_i),  N_i = eta_i / max(|eta_i|, EPS)
"""
from __future__ import annotations

import numpy as np

import ref64
from ref64 import EPS, R64


def cross_abs(a, b):
    """componentwise bound of |a x b| from |a| and |b| (the size of the two products each component is formed from)"""
    return np.stack([a[:, 1] * b[:, 2] + a[:, 2] * b[:, 1],
                     a[:, 2] * b[:, 0] + a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] + a[:, 1] * b[:, 0]], 1)


def moment(P, rho0):
    """M_i = sum_j V_j g(r) d d^T with gradW_ij = g(r) d (fluid pairs): (n, 3, 3)"""
    G = ref64.grad_W(P.dF, P.rF, P.R)[0]
    t = (P.mF / rho0)[:, None, None] * P.dF[:, :, None] * G[:, None, :]
    M = np.zeros((P.n, 3, 3))
    np.add.at(M, P.iF, t)
    return M


def vorticity(P, vel, rho0):
    """(omega R64 (n, 3), |omega| R64 (n,))"""
    vel = np.asarray(vel, np.float64)
    gv, gs = ref64.grad_W(P.dF, P.rF, P.R)
    u = vel[P.iF] - vel[P.jF]
    V = P.mF / rho0
    w, m = P.sum2((V[:, None] * np.cross(u, gv), V[:, None] * cross_abs(np.abs(u), gs)))
    return R64(w, m), R64(np.sqrt((w ** 2).sum(1)), np.sqrt((m ** 2).sum(1)))


def eta(P, omega_norm, rho0):
    """eta R64 (n, 3), difference form"""
    wn = np.asarray(omega_norm, np.float64)
    gv, gs = ref64.grad_W(P.dF, P.rF, P.R)
    c = (P.mF / rho0) * (wn[P.jF] - wn[P.iF])
    return R64(*P.sum2(ref64.mul(c, (gv, gs))))


def vorticity_confinement(P, omega, omega_norm, eps, dt, rho0):
    """(dv R64 (n, 3), eta R64): dv's mag carries the error of N = eta / |eta| (relative 2 tau mag_eta / |eta|, meaningful
    where eta is well conditioned) and the rounding of the cross product"""
    w = np.asarray(omega, np.float64)
    e = eta(P, omega_norm, rho0)
    le = np.sqrt((e.value ** 2).sum(1))
    N = e.value / np.maximum(le, EPS)[:, None]
    dv = dt * eps * np.cross(N, w)
    lw = np.sqrt((w ** 2).sum(1))
    me = np.sqrt((e.mag ** 2).sum(1))
    cond = 2.0 * me / np.maximum(le, EPS)
    mag = dt * eps * (lw * cond)[:, None] + dt * eps * cross_abs(np.abs(N), np.abs(w))
    return R64(dv, mag), e


def well_conditioned(e: R64, tau, floor=0.0):
    """particles whose eta direction is determined: |eta| >= 100 (tau |mag_eta| + floor)"""
    le = np.sqrt((e.value ** 2).sum(1))
    me = np.sqrt((e.mag ** 2).sum(1))
    return le >= 100.0 * (tau * me + floor)
