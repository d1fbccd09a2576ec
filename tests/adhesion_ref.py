"""Float64 reference of fluid-solid adhesion (DESIGN.md section 2.11) -- TEST INFRASTRUCTURE ONLY (numpy).

From the fluid-boundary pairs of ref64.Pairs (d = x_i - x_b, r = |d|):
    a_i = - sum_b beta_g(b) Psi_b A(r) d / r,   Psi_b = rho0 m_b / rho_B
    A(r) = 0.007 / R^3.25 (-4 r^2 / R + 6 r - 2 R)^(1/4)   for R/2 < r <= R, else 0
The fourth root makes A steep at r = R/2: a float32 r, formed from float32 positions and so off by a few ulp of the coordinates, moves A
there by far more than its own rounding, and a pair within that error of either end of the band may fall on either side.  `mag` carries
both: each pair's size is its term times (1 + the relative change of A / r under the distance error dr, over ref64.TAU), and a pair within 2 dr of an end counts
with the term it would have just inside.
"""
from __future__ import annotations

import numpy as np

import ref64


def distance_error(pos):
    """the error of a float32 distance between float32 positions of this size: a few ulp of the largest coordinate"""
    return 4.0 * float(np.spacing(np.float32(np.abs(np.asarray(pos, np.float32)).max())))


def kernel(r, R):
    """A(r); zero outside (R/2, R]"""
    r = np.asarray(r, np.float64)
    t = -4.0 * r * r / R + 6.0 * r - 2.0 * R
    inside = (2.0 * r > R) & (r <= R)
    return np.where(inside, 0.007 / R ** 3.25 * np.maximum(t, 0.0) ** 0.25, 0.0)


def _group_beta(P, beta, groups):
    """beta of each fluid-boundary pair's group (groups: the boundary group of every boundary slot, None: all walls)"""
    beta = np.asarray(beta, np.float64)
    g = np.zeros(P.jB.size, np.int64) if groups is None else np.asarray(groups, np.int64)[P.jB]
    b = np.zeros(P.jB.size)
    ok = g < beta.size
    b[ok] = beta[g[ok]]
    return b


def accel(P, beta, rho0, rhoB, groups=None, dr=0.0, off=None):
    """a_i as ref64.R64, and the bounds {lo, hi} of the wetted count; dr: the absolute error of a float32 distance
    (distance_error of the positions); off: fluid particles off the grid, which do not interact (zero rows, not counted)"""
    R = P.R
    r = P.rB
    bp = _group_beta(P, beta, groups)
    if off is not None:
        bp = np.where(np.asarray(off)[P.iB], 0.0, bp)
    lo_edge, hi_edge = 0.5 * R + 2.0 * dr, R - 2.0 * dr
    near = ((r > 0.5 * R - 2.0 * dr) & (r <= lo_edge)) | ((r > hi_edge) & (r <= R + 2.0 * dr))
    rr = np.clip(r, lo_edge, hi_edge)
    A = kernel(r, R)
    Anear = kernel(rr, R)
    t = -4.0 * rr * rr / R + 6.0 * rr - 2.0 * R
    sens = (0.25 * np.abs(6.0 - 8.0 * rr / R) / np.maximum(t, 1e-300) + 1.0 / rr) * dr
    psi = rho0 * P.mB / rhoB
    c = bp * psi * A / np.where(r > 0, r, 1.0)
    cn = bp * psi * Anear / np.where(r > 0, r, 1.0)
    term = -c[:, None] * P.dB
    size = np.abs(c)[:, None] * np.abs(P.dB) * (1.0 + sens / ref64.TAU)[:, None]     # (the check allows TAU * mag)
    size = np.where(near[:, None], np.abs(cn)[:, None] * np.abs(P.dB) / ref64.TAU, size)
    v, m = P.sum(P.iB, (term, size))
    sure = (bp > 0) & (r > lo_edge) & (r <= hi_edge)
    maybe = (bp > 0) & (A > 0) | (bp > 0) & near
    lo = np.unique(P.iB[sure]).size
    hi = np.unique(P.iB[maybe]).size
    return ref64.R64(v, m), lo, hi


def reaction(P, beta, rho0, rhoB, dt, massF, posB, groups, centres):
    """{J, H} of every body (rows 0..): the impulse dt m_i beta_g Psi_k A d / r on body particle k and its moment about the centre"""
    bp = _group_beta(P, beta, groups)
    g = np.asarray(groups, np.int64)[P.jB]
    A = kernel(P.rB, P.R)
    psi = rho0 * P.mB / rhoB
    f = (dt * np.asarray(massF, np.float64)[P.iB] * bp * psi * A / np.where(P.rB > 0, P.rB, 1.0))[:, None] * P.dB
    centres = np.asarray(centres, np.float64)
    out = np.zeros((centres.shape[0], 6))
    for k in range(centres.shape[0]):
        sel = g == k + 1
        arm = np.asarray(posB, np.float64)[P.jB[sel]] - centres[k]
        out[k, :3] = f[sel].sum(0)
        out[k, 3:] = np.cross(arm, f[sel]).sum(0)
    return out
