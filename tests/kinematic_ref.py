"""float64 reference of the kinematic rigid bodies (DESIGN.md section 2.3): pose update, placement, per-group boundary
masses, and the DFSPH divergence sums with boundary velocities.  numpy + scipy only.

Poses are {c, q = (x, y, z, w)} (scalar part last), motions {V, Omega} in the world frame, as in include/sphk.h."""
import numpy as np
from scipy.spatial import cKDTree

import ref64


def quat_mul(a, b):
    """Hamilton product a (x) b of (x, y, z, w) quaternions"""
    av, aw, bv, bw = a[:3], a[3], b[:3], b[3]
    return np.concatenate([aw * bv + bw * av + np.cross(av, bv), [aw * bw - av @ bv]])


def rotation(q):
    """R(q) of a unit (x, y, z, w) quaternion"""
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose_update(pose, motion, dt):
    """c <- c + dt V; q <- normalize(dq (x) q), dq the rotation by |Omega| dt about Omega (identity for Omega = 0)"""
    pose, motion = np.asarray(pose, np.float64), np.asarray(motion, np.float64)
    c = pose[:3] + dt * motion[:3]
    q = pose[3:7]
    W = motion[3:6]
    w = np.linalg.norm(W)
    if w > 0.0:
        h = 0.5 * w * dt
        q = quat_mul(np.concatenate([np.sin(h) * W / w, [np.cos(h)]]), q)
        q = q / np.linalg.norm(q)
    return np.concatenate([c, q])


def place(pose, motion, r):
    """x_k = c + R(q) r_k, v_k = V + Omega x (x_k - c)"""
    pose, motion, r = (np.asarray(a, np.float64) for a in (pose, motion, r))
    d = r @ rotation(pose[3:7]).T
    return pose[:3] + d, motion[:3] + np.cross(motion[3:6], d)


def grouped_masses(posB, group, rhoB, R):
    """m_b = rhoB / max(eps, sum over b's group of W_bk) (the static set is group 0, body b is group b + 1)"""
    posB = np.asarray(posB, np.float64)
    group = np.asarray(group)
    n = posB.shape[0]
    m = np.zeros(n)
    for g in np.unique(group):
        idx = np.nonzero(group == g)[0]
        pts = posB[idx]
        pr = cKDTree(pts).sparse_distance_matrix(cKDTree(pts), R * (1.0 + 1e-6), output_type="ndarray")
        r = np.sqrt(((pts[pr["i"]] - pts[pr["j"]]) ** 2).sum(1))
        s = np.bincount(pr["i"], ref64.W(r, R)[0], len(idx))
        m[idx] = rhoB / np.maximum(ref64.EPS, s)
    return m


def divergence(P, vel, velB):
    """sum_j m_j (v_i - v_j) . gradW_ij over fluid and boundary neighbours, with the boundary velocities v_b (ref64's
    _divergence is the case v_b = 0)"""
    vel, velB = np.asarray(vel, np.float64), np.asarray(velB, np.float64)
    tF = ref64.mul(P.mF, ref64.dot(vel[P.iF] - vel[P.jF], ref64.grad_W(P.dF, P.rF, P.R)))
    tB = ref64.mul(P.mB, ref64.dot(vel[P.iB] - velB[P.jB], ref64.grad_W(P.dB, P.rB, P.R)))
    return P.sum2(tF, tB)


def dfsph_div_error(P, vel, velB, dens, alpha, dt, rho0, tau):
    """ref64.dfsph_div_error with boundary velocities"""
    dens, alpha = np.asarray(dens, np.float64), np.asarray(alpha, np.float64)
    e, m = divergence(P, vel, velB)
    e = np.maximum(0.0, e)
    below = dens <= rho0
    zero = (dens + dt * e < rho0) & below
    val = np.where(zero, 0.0, e)
    near = below & (np.abs(dens + dt * e - rho0) <= dt * tau * m + 2.0 * float(np.spacing(np.float32(rho0))))
    alt = np.where(near, np.where(zero, e, 0.0), val)
    return ref64.R64(val, m, alt), ref64.R64(val * alpha, m * np.abs(alpha), alt * alpha)


def dfsph_den_error(P, vel, velB, dens, alpha, dt, rho0):
    """ref64.dfsph_den_error with boundary velocities"""
    dens, alpha = np.asarray(dens, np.float64), np.asarray(alpha, np.float64)
    s, m = divergence(P, vel, velB)
    e = np.maximum(0.0, dt * s + dens - rho0)
    me = dt * m
    fe = ref64.f32_spacing(np.abs(dens) + me) + ref64.f32_spacing(e)
    k = e * alpha
    return ref64.R64(e, me, floor=fe), ref64.R64(k, me * np.abs(alpha), floor=fe * np.abs(alpha) + ref64.f32_spacing(k))
