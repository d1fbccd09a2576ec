"""A float64 reference of the implicit viscosity solve (DESIGN.md section 2.5) -- TEST INFRASTRUCTURE ONLY (numpy + scipy).

From the explicit pair lists of ref64.Pairs (or any object with the same fields) it forms, per element with the magnitude
the ref64 bounds use, the two sweeps of the solve:
    c_ij    = -10 nu V_j g(r) / (r^2 + 0.01 R^2),  V_j = m_j / rho0     (boundary: nu_b, m_b / rho_B)
    D_i     = I + dt sum_j c_ij d d^T + dt sum_b c_ib d d^T              (as {xx, yy, zz, xy, xz, yz})
    b_i     = v*_i + dt sum_b c_ib d (d . v_b)
    (A p)_i = D_i p_i - dt sum_j c_ij d (d . p_j)
assembles A as a scipy.sparse matrix, solves A v = b exactly, and runs the engine's PCG (x0 = v*, mass inner product,
block-Jacobi preconditioner, the same loop test) in float64.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps
import scipy.sparse.linalg as spl

import ref64

SYM = ((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2))      # the 6-float layout of a symmetric 3x3


def grad_factor(r, R):
    """the kernel gradient factor g (gradW = g d) and the size of its float32 operands (ref64.grad_W's)"""
    q = 2.0 * r / R
    outer = q > 1.0
    s = np.where(outer, (12.0 - 3.0 * q) * q - 12.0, (9.0 * q - 12.0) * q)
    ss = np.where(outer, (12.0 + 3.0 * q) * q + 12.0, (9.0 * q + 12.0) * q)
    c = np.where(q > 2.0, 0.0, 1.0 / (np.pi * (q + ref64.EPS) * R ** 5))
    return s * c, ss * c


def coefficients(P, nu, nu_b, rho0, rho_b):
    """(c, size of c) of the fluid pairs and of the boundary pairs"""
    den = lambda r: r * r + 0.01 * P.R * P.R  # noqa: E731
    g, gs = grad_factor(P.rF, P.R)
    gb, gbs = grad_factor(P.rB, P.R)
    vF, vB = nu * P.mF / rho0, nu_b * P.mB / rho_b
    return (-10.0 * vF * g / den(P.rF), 10.0 * vF * gs / den(P.rF)), (-10.0 * vB * gb / den(P.rB), 10.0 * vB * gbs / den(P.rB))


def _outer_sum(P, i, d, c):
    """sum over the pairs of each particle of c d d^T, as (n, 3, 3)"""
    out = np.zeros((P.n, 3, 3))
    for a in range(3):
        for b in range(3):
            out[:, a, b] = np.bincount(i, c * d[:, a] * d[:, b], P.n)
    return out


def setup(P, vel, vel_b, nu, nu_b, dt, rho0, rho_b):
    """(D as (n, 3, 3), mag of D, b, mag of b) of OpViscImplicitSetup; vel_b = the boundary records' velocities"""
    (cF, sF), (cB, sB) = coefficients(P, nu, nu_b, rho0, rho_b)
    S = _outer_sum(P, P.iF, P.dF, cF) + _outer_sum(P, P.iB, P.dB, cB)
    mS = _outer_sum(P, P.iF, np.abs(P.dF), sF) + _outer_sum(P, P.iB, np.abs(P.dB), sB)
    D = np.eye(3)[None] + dt * S
    vb = np.asarray(vel_b, np.float64)[P.jB]
    dvb = (P.dB * vb).sum(1)
    sdvb = (np.abs(P.dB) * np.abs(vb)).sum(1)
    bt = np.stack([np.bincount(P.iB, cB * dvb * P.dB[:, k], P.n) for k in range(3)], 1)
    bm = np.stack([np.bincount(P.iB, sB * sdvb * np.abs(P.dB[:, k]), P.n) for k in range(3)], 1)
    b = np.asarray(vel, np.float64) + dt * bt
    return D, dt * mS, b, dt * bm


def packed(D):
    """(n, 3, 3) -> (n, 6) in the engine's layout"""
    return np.stack([D[:, a, b] for a, b in SYM], 1)


def unpacked(D6):
    D6 = np.asarray(D6, np.float64)
    out = np.zeros((D6.shape[0], 3, 3))
    for k, (a, b) in enumerate(SYM):
        out[:, a, b] = out[:, b, a] = D6[:, k]
    return out


def matvec(P, D, p, nu, dt, rho0):
    """((A p), mag) of OpViscImplicitMatvec with the given D (n, 3, 3)"""
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


def assemble(P, nu, nu_b, dt, rho0, rho_b):
    """A (3n x 3n, CSR) and D (n, 3, 3); D from the boundary pairs' coefficients too"""
    (cF, _), (cB, _) = coefficients(P, nu, nu_b, rho0, rho_b)
    D = np.eye(3)[None] + dt * (_outer_sum(P, P.iF, P.dF, cF) + _outer_sum(P, P.iB, P.dB, cB))
    rows, cols, vals = [], [], []
    ii = np.arange(P.n)
    for a in range(3):
        for b in range(3):
            rows += [3 * ii + a, 3 * P.iF + a]
            cols += [3 * ii + b, 3 * P.jF + b]
            vals += [D[:, a, b], -dt * cF * P.dF[:, a] * P.dF[:, b]]
    A = sps.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * P.n, 3 * P.n))
    return A, D


def solve(A, b):
    """the exact solution of A v = b, (n, 3)"""
    return spl.spsolve(A.tocsc(), np.asarray(b, np.float64).ravel()).reshape(-1, 3)


def pcg(A, D, b, x0, mass, tol, max_iter, precond="block", weighted=True):
    """The engine's PCG in float64: (x, iterations, |r|_M / |b|_M of the recursive residual).  precond: "block" (D_i^-1) or
    "diag" (the diagonal of D_i only); weighted=False: Euclidean dot products instead of the mass inner product (the two
    variants exist to show that a scene tells them apart)."""
    m3 = np.repeat(np.asarray(mass, np.float64) if weighted else np.ones(len(mass)), 3)
    Dinv = np.linalg.inv(D) if precond == "block" else np.stack([np.diag(1.0 / np.diagonal(x)) for x in D])
    dot = lambda u, w: float((m3 * u * w).sum())  # noqa: E731
    prec = lambda r: np.einsum("nab,nb->na", Dinv, r.reshape(-1, 3)).ravel()  # noqa: E731
    b = np.asarray(b, np.float64).ravel()
    x = np.asarray(x0, np.float64).ravel().copy()
    r = b - A @ x
    z = prec(r)
    p = z.copy()
    bb, rz, rr = dot(b, b), dot(r, z), dot(r, r)
    it = 0
    tol2 = float(tol) ** 2
    if not (rr <= tol2 * bb or rz == 0.0):
        while True:
            Ap = A @ p
            pAp = dot(p, Ap)
            if not pAp > 0.0:
                break
            alpha = rz / pAp
            x += alpha * p
            r -= alpha * Ap
            z = prec(r)
            rzn, rr = dot(r, z), dot(r, r)
            it += 1
            if rr <= tol2 * bb or rzn == 0.0 or it >= max_iter:
                break
            p = z + (rzn / rz) * p
            rz = rzn
    return x.reshape(-1, 3), it, (np.sqrt(rr / bb) if bb > 0 else 0.0)


def m_norm(v, mass):
    v = np.asarray(v, np.float64)
    return float(np.sqrt((np.asarray(mass, np.float64)[:, None] * v * v).sum()))


def spectrum(A, mass, which):
    """the largest ("LA") or smallest ("SA") eigenvalue of A (self-adjoint in the mass inner product): of M^1/2 A M^-1/2"""
    s = np.sqrt(np.repeat(np.asarray(mass, np.float64), 3))
    S = sps.diags(s) @ A @ sps.diags(1.0 / s)
    S = 0.5 * (S + S.T)
    return float(spl.eigsh(S, k=1, which=which, return_eigenvectors=False, tol=1e-10)[0])
