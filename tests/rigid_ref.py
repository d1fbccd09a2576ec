"""Float64 reference of two-way coupled rigid bodies (DESIGN.md section 2.4): the fluid's reaction on body particles from
explicit pair lists, the end-of-step Newton-Euler update and the wall contact.  Conventions of ref64 / kinematic_ref:
quaternions (x, y, z, w), motions {V, Omega} in the world frame, d = x_i - x_k."""
import numpy as np
from scipy.spatial import cKDTree

import ref64
from kinematic_ref import rotation


def reaction(xf, sf, mf, xb, mb, group, centres, coef, R):
    """{J, H} per body (n_bodies, 6) and the sum of |terms| per component (mag) of one reacting sweep: the fluid particle i
    receives coef m_i m_k s_i gradW(x_i - x_k); body particle k of body group[k] gathers the opposite and its moment about
    centres[group[k]].  xf, sf, mf: fluid positions, record scalars, masses; xb, mb: body particles and masses."""
    xf, xb = np.asarray(xf, np.float64), np.asarray(xb, np.float64)
    n_bodies = len(centres)
    out, mag = np.zeros((n_bodies, 6)), np.zeros((n_bodies, 6))
    pairs = cKDTree(xb).query_ball_tree(cKDTree(xf), R * (1.0 + 1e-5))
    k = np.repeat(np.arange(len(xb)), [len(p) for p in pairs])
    i = np.fromiter((j for p in pairs for j in p), np.int64, count=len(k))
    if len(k) == 0:
        return out, mag
    d = xf[i] - xb[k]
    g, gs = ref64.grad_W(d, np.linalg.norm(d, axis=1), R)
    w = (-coef * np.asarray(mf, np.float64)[i] * np.asarray(mb, np.float64)[k] * np.asarray(sf, np.float64)[i])[:, None]
    f, fs = w * g, np.abs(w) * gs
    r = xb[k] - np.asarray(centres, np.float64)[group[k]]
    t = np.cross(r, f)
    ts = np.abs(r[:, [1, 2, 0]]) * fs[:, [2, 0, 1]] + np.abs(r[:, [2, 0, 1]]) * fs[:, [1, 2, 0]]
    for b in range(n_bodies):
        m = group[k] == b
        out[b, :3], out[b, 3:] = f[m].sum(0), t[m].sum(0)
        mag[b, :3], mag[b, 3:] = fs[m].sum(0), ts[m].sum(0)
    return out, mag


def world_inertia(q, inertia):
    R = rotation(q)
    return R @ np.diag(np.asarray(inertia, np.float64)) @ R.T


def integrate(motion, q, mass, inertia, J, H, dt, G):
    """end of step of a dynamic body: V += J/M + dt G; L = Iw Omega + H; Omega = Iw^-1 L (Iw from the current q)"""
    motion = np.asarray(motion, np.float64)
    V = motion[:3] + np.asarray(J, np.float64) / mass + dt * np.asarray(G, np.float64)
    Iw = world_inertia(q, inertia)
    W = np.linalg.solve(Iw, Iw @ motion[3:] + np.asarray(H, np.float64))
    return np.concatenate([V, W])


def contact(c, q, V, box_lo, box_hi, clamp_hi):
    """wall contact after the pose update: the corners of the body-frame box [box_lo, box_hi] at pose (c, q) are pushed
    back into [0, clamp_hi] per axis by moving the centre; the outward velocity component is zeroed"""
    c, V = np.array(c, np.float64), np.array(V, np.float64)
    lo, hi = np.asarray(box_lo, np.float64), np.asarray(box_hi, np.float64)
    corners = np.array([[(hi if s & 1 else lo)[0], (hi if s & 2 else lo)[1], (hi if s & 4 else lo)[2]] for s in range(8)])
    x = c + corners @ rotation(q).T
    for a in range(3):
        if x[:, a].min() < 0.0:
            c[a] -= x[:, a].min()
            V[a] = max(V[a], 0.0)
        elif x[:, a].max() > clamp_hi[a]:
            c[a] -= x[:, a].max() - clamp_hi[a]
            V[a] = min(V[a], 0.0)
    return c, V
