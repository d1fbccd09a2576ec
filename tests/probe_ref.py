"""A float64 reference of the probes and water-level gauges (DESIGN.md section 2.13) -- TEST INFRASTRUCTURE ONLY (numpy + scipy).

For a point x, over the counted fluid particles j (in the grid, rho_j > 0) with |x - x_j| <= R, V_j = m_j / rho_j and the continuous
cubic spline W (no quirk Q1):  S = sum V_j W,  A = sum V_j A_j W / S  for A in {rho, v, p, T}.  Pairs come from cKDTree, so the
reference knows nothing of cells or reach.  Every output comes with `mag`, a bound on the sum of the sizes of its float32 terms, so
that a float32 implementation that forms the same sums in any order is within

    |x - value| <= tau * mag + floor

element by element.  A term's size is V_j (W_j + 4 cW): the second part covers the rounding of q = r / h near the support edge,
where W is tiny but its float32 value carries the absolute error of (2 - q)^3.  A quotient A = N / S carries
mag_A = (sum |size_j A_j|) / S + |A| (sum size_j) / S.  n is compared against the counts at R (1 - 1e-6) and R (1 + 1e-6).
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

F = np.float32
TAU = 1e-5          # the per-element bound of the float32 probe kernels (largest observed ratios: DESIGN.md section 2.13)


def cW(R):
    return 0.25 / (np.pi * R ** 3)


def W(r, R):
    """the continuous cubic spline of support R (W(0) = 4 cW, W(R) = 0)"""
    q = 2.0 * np.asarray(r, np.float64) / R
    w = np.where(q > 1.0, (2.0 - q) ** 3, (3.0 * q - 6.0) * q * q + 4.0)
    return np.where(q > 2.0, 0.0, cW(R) * w)


def records(points, pos, vel, mass, density, R, counted=None, point_dry=None, pressure=None, temperature=None):
    """value (P, 8), mag (P, 8), n_lo (P,), n_hi (P,) of the records {S, rho, vx, vy, vz, p, T, n}.  counted: bool mask of the
    particles that take part (default all); point_dry: bool mask of points outside the grid (forced dry)."""
    x = np.asarray(points, np.float64).reshape(-1, 3)
    P = x.shape[0]
    pos = np.asarray(pos, np.float64)
    rho = np.asarray(density, np.float64)
    ok = (rho > 0) if counted is None else (np.asarray(counted, bool) & (rho > 0))
    idx = np.nonzero(ok)[0]
    value, mag = np.zeros((P, 8)), np.zeros((P, 8))
    n_lo, n_hi = np.zeros(P, np.int64), np.zeros(P, np.int64)
    value[:, 5] = np.nan if pressure is None else 0.0
    value[:, 6] = np.nan if temperature is None else 0.0
    if idx.size == 0 or P == 0:
        return value, mag, n_lo, n_hi
    tree = cKDTree(pos[idx])
    lists = tree.query_ball_point(x, R * (1.0 + 1e-6))
    V = np.asarray(mass, np.float64)[idx] / rho[idx]
    fields = [rho[idx], *np.asarray(vel, np.float64)[idx].T]
    fields.append(np.asarray(pressure, np.float64)[idx] if pressure is not None else None)
    fields.append(np.asarray(temperature, np.float64)[idx] if temperature is not None else None)
    for k in range(P):
        if point_dry is not None and point_dry[k]:
            continue
        js = np.asarray(lists[k], np.int64)
        if js.size == 0:
            continue
        r = np.sqrt(((x[k] - pos[idx][js]) ** 2).sum(1))
        n_hi[k] = js.size
        n_lo[k] = int(np.count_nonzero(r <= R * (1.0 - 1e-6)))
        inside = r <= R
        w = W(r, R) * inside
        vw = V[js] * w
        size = V[js] * (w + 4.0 * cW(R))
        S = vw.sum()
        value[k, 0], mag[k, 0] = S, size.sum()
        value[k, 7] = np.count_nonzero(inside)
        if not S > 0:
            continue
        for f, a in enumerate(fields):
            col = 1 + f
            if a is None:
                continue
            A = (vw * a[js]).sum() / S
            value[k, col] = A
            mag[k, col] = (size * np.abs(a[js])).sum() / S + abs(A) * size.sum() / S
    return value, mag, n_lo, n_hi


def gauge_points(a, b, k):
    """the k sample points of a gauge, in the float32 operations of the kernel: a + (b - a) * (i / (k - 1)), each rounded once"""
    a, b = np.asarray(a, F), np.asarray(b, F)
    t = (np.arange(k, dtype=F) / F(k - 1)).astype(F)
    return (a[None, :] + ((b - a)[None, :] * t[:, None]).astype(F)).astype(F)


def level_from_profile(S, theta, L, mag=None, tau=TAU):
    """(level, bound, ambiguous) of a gauge from its S profile (float64): the linear crossing of theta between the highest wet
    sample i* and i* + 1, times L / (k - 1); L when i* = k - 1; -1 when dry.  ambiguous: some sample lies within tau * mag of theta,
    so a float32 profile may pick another i*."""
    S = np.asarray(S, np.float64)
    k = S.size
    ambiguous = mag is not None and bool(np.any(np.abs(S - theta) <= tau * np.asarray(mag) + 1e-12))
    wet = np.nonzero(S >= theta)[0]
    if wet.size == 0:
        return -1.0, 0.0, ambiguous
    i = int(wet[-1])
    if i == k - 1:
        return float(L), 1e-6 * L, ambiguous
    d = S[i] - S[i + 1]
    f = (S[i] - theta) / d
    bound = 1e-6 * L
    if mag is not None:
        bound += L / (k - 1) * tau * (mag[i] + mag[i + 1]) * (1.0 + abs(f)) / d
    return L * (i + f) / (k - 1), bound, ambiguous


def gauge_levels(gauges, theta, pos, mass, density, R, counted=None, dry_of=None):
    """[(level, bound, ambiguous)] of (a, b, k) gauges; dry_of(points) -> bool mask of points outside the grid"""
    out = []
    for a, b, k in gauges:
        pts = gauge_points(a, b, k)
        v, m, _, _ = records(pts, pos, np.zeros_like(np.asarray(pos)), mass, density, R, counted,
                             None if dry_of is None else dry_of(pts))
        d = np.asarray(b, F).astype(np.float64) - np.asarray(a, F).astype(np.float64)
        out.append(level_from_profile(v[:, 0], theta, float(np.sqrt((d ** 2).sum())), m[:, 0]))
    return out
