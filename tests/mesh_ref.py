"""Float64 reference of the mesh scene builders (DESIGN.md section 2.12) and the test meshes.

  winding_number   generalized winding number (sum of signed solid angles / 4 pi, Van Oosterom and Strackee): 1 inside a closed,
                   outward-wound mesh, 0 outside, independent of any ray
  distance         exact point-triangle distance (closest point by region), minimum over all triangles
  mass_properties  volume, centroid and inertia per unit density about the centroid by the divergence theorem (tetrahedra from
                   the origin), straight from the polyhedral formulas
The meshes are generated here: box, icosphere, torus, an open plate and an L-shaped prism, all counter-clockwise from outside."""
import numpy as np


# ---- meshes --------------------------------------------------------------------------------------------------------------------
def box(lo, hi):
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    v = np.array([[lo[0] if i & 1 == 0 else hi[0], lo[1] if i & 2 == 0 else hi[1], lo[2] if i & 4 == 0 else hi[2]] for i in range(8)])
    f = np.array([[0, 2, 3], [0, 3, 1], [4, 5, 7], [4, 7, 6], [0, 1, 5], [0, 5, 4], [2, 6, 7], [2, 7, 3], [0, 4, 6], [0, 6, 2],
                  [1, 3, 7], [1, 7, 5]])
    return v, f


def icosphere(subdiv, radius=1.0, center=(0.0, 0.0, 0.0)):
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t], [t, 0, -1], [t, 0, 1],
         [-t, 0, -1], [-t, 0, 1]]
    v = [list(np.asarray(p) / np.linalg.norm(p)) for p in v]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
         [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    for _ in range(subdiv):
        mid = {}

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = (np.asarray(v[a]) + np.asarray(v[b])) / 2.0
                v.append(list(p / np.linalg.norm(p)))
                mid[k] = len(v) - 1
            return mid[k]
        nf = []
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return np.asarray(v) * radius + np.asarray(center), np.asarray(f)


def torus(R, r, nu=32, nv=16, center=(0.0, 0.0, 0.0)):
    """axis along y"""
    u, w = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    v = np.stack([(R + r * np.cos(w)) * np.cos(u), r * np.sin(w), (R + r * np.cos(w)) * np.sin(u)], -1).reshape(-1, 3)
    f = []
    for i in range(nu):
        for j in range(nv):
            a, b, c, d = i * nv + j, ((i + 1) % nu) * nv + j, ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
            f += [[a, c, b], [a, d, c]]
    return v + np.asarray(center), np.asarray(f)


def plate(lo, hi, y, n=4):
    """an open, horizontal n x n plate at height y (normal +y)"""
    xs, zs = np.linspace(lo[0], hi[0], n + 1), np.linspace(lo[1], hi[1], n + 1)
    v = np.array([[x, y, z] for x in xs for z in zs])
    f = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1, i * (n + 1) + j + 1
            f += [[a, d, c], [a, c, b]]
    return v, np.asarray(f)


def l_prism(o, a, depth):
    """an L-shaped prism: the L (2a x 2a without the a x a upper right square) in (x, y), extruded along z from o"""
    L = np.array([[0, 0], [2 * a, 0], [2 * a, a], [a, a], [a, 2 * a], [0, 2 * a]], np.float64)
    n = len(L)
    v = np.concatenate([np.c_[L, np.zeros(n)], np.c_[L, np.full(n, depth)]]) + np.asarray(o)
    f = [[0, 2, 1], [0, 3, 2], [0, 5, 3], [5, 4, 3]]                    # back (z = 0), seen from -z
    f += [[n + 0, n + 1, n + 2], [n + 0, n + 2, n + 3], [n + 0, n + 3, n + 5], [n + 5, n + 3, n + 4]]
    for k in range(n):
        j = (k + 1) % n
        f += [[k, j, n + j], [k, n + j, n + k]]
    return v, np.asarray(f)


def write_obj(path, v, f):
    with open(path, "w") as fh:
        for p in v:
            fh.write("v %r %r %r\n" % tuple(float(np.float32(x)) for x in p))
        for t in f:
            fh.write("f %d %d %d\n" % tuple(int(i) + 1 for i in t))
    return str(path)


# ---- queries -------------------------------------------------------------------------------------------------------------------
def winding_number(p, v, f, chunk=4096):
    p = np.asarray(p, np.float64)
    A, B, C = (np.asarray(v, np.float64)[np.asarray(f)[:, k]] for k in range(3))
    out = np.zeros(len(p))
    for s in range(0, len(p), chunk):
        q = p[s:s + chunk, None, :]
        a, b, c = A[None] - q, B[None] - q, C[None] - q
        la, lb, lc = (np.linalg.norm(x, axis=-1) for x in (a, b, c))
        det = np.einsum("...i,...i", a, np.cross(b, c))
        den = la * lb * lc + np.einsum("...i,...i", a, b) * lc + np.einsum("...i,...i", b, c) * la + np.einsum("...i,...i", c, a) * lb
        out[s:s + chunk] = np.arctan2(det, den).sum(1) / (2 * np.pi)
    return out


def _closest(p, a, b, c):
    """closest points on triangles (broadcast): Ericson, Real-Time Collision Detection 5.1.5, in float64"""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = (ab * ap).sum(-1), (ac * ap).sum(-1)
    bp = p - b
    d3, d4 = (ab * bp).sum(-1), (ac * bp).sum(-1)
    cp = p - c
    d5, d6 = (ab * cp).sum(-1), (ac * cp).sum(-1)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    with np.errstate(divide="ignore", invalid="ignore"):
        den = va + vb + vc
        q = a + ab * (vb / den)[..., None] + ac * (vc / den)[..., None]
        e_ab = a + ab * (d1 / (d1 - d3))[..., None]
        e_ac = a + ac * (d2 / (d2 - d6))[..., None]
        e_bc = b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[..., None]
    q = np.where(((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0))[..., None], e_bc, q)
    q = np.where(((vb <= 0) & (d2 >= 0) & (d6 <= 0))[..., None], e_ac, q)
    q = np.where(((d6 >= 0) & (d5 <= d6))[..., None], c, q)
    q = np.where(((vc <= 0) & (d1 >= 0) & (d3 <= 0))[..., None], e_ab, q)
    q = np.where(((d3 >= 0) & (d4 <= d3))[..., None], b, q)
    q = np.where(((d1 <= 0) & (d2 <= 0))[..., None], a, q)
    return q


def distance(p, v, f, chunk=1024):
    p = np.asarray(p, np.float64)
    A, B, C = (np.asarray(v, np.float64)[np.asarray(f)[:, k]] for k in range(3))
    out = np.empty(len(p))
    for s in range(0, len(p), chunk):
        q = p[s:s + chunk, None, :]
        out[s:s + chunk] = np.sqrt(((_closest(q, A[None], B[None], C[None]) - q) ** 2).sum(-1).min(1))
    return out


def mass_properties(v, f):
    """(V, centroid, inertia 3x3 per unit density about the centroid) of a closed, outward-wound mesh"""
    v = np.asarray(v, np.float64)
    a, b, c = (v[np.asarray(f)[:, k]] for k in range(3))
    D = np.einsum("ij,ij->i", a, np.cross(b, c))
    s = a + b + c
    V = D.sum() / 6.0
    m1 = (D[:, None] * s).sum(0) / 24.0
    m2 = np.einsum("t,ti,tj->ij", D, s, s) + sum(np.einsum("t,ti,tj->ij", D, x, x) for x in (a, b, c))
    m2 /= 120.0
    cen = m1 / V
    Cm = m2 - V * np.outer(cen, cen)
    return V, cen, np.trace(Cm) * np.eye(3) - Cm


def area(v, f):
    v = np.asarray(v, np.float64)
    a, b, c = (v[np.asarray(f)[:, k]] for k in range(3))
    return 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum()


def surface_points(v, f, h):
    """float64 points on every triangle at spacing <= h (a barycentric lattice), for coverage checks"""
    v = np.asarray(v, np.float64)
    out = []
    for t in np.asarray(f):
        a, b, c = v[t]
        m = max(1, int(np.ceil(max(np.linalg.norm(b - a), np.linalg.norm(c - b), np.linalg.norm(a - c)) / h)))
        i, j = np.meshgrid(np.arange(m + 1), np.arange(m + 1), indexing="ij")
        k = i + j <= m
        i, j = i[k] / m, j[k] / m
        out.append(a + i[:, None] * (b - a) + j[:, None] * (c - a))
    return np.concatenate(out)
