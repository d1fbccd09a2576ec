"""Float64 reference of the mesh scene builders (DESIGN.md section 2.12) and the test meshes.

  winding_number   generalized winding number (sum of signed solid angles / 4 pi, Van Oosterom and Strackee): 1 inside a closed,
                   outward-wound mesh, 0 outside, independent of any ray
  distance         exact point-triangle distance (closest point by region), minimum over all triangles
  mass_properties  volume, centroid and inertia per unit density about the centroid by the divergence theorem (tetrahedra from
                   the origin), straight from the polyhedral formulas
  lattice          the points sphk_mesh_fill forms, in its order, over the index ranges it computes (fill_ranges)
  sphere_gap, torus_gap, sphere_band, torus_band
                   signed distance to the ideal sphere or torus and a bound on how far the mesh's facets stray from it, for
                   inside and distance tests on meshes too large for the O(points x triangles) queries
The meshes are generated here: box, icosphere, torus, an open plate and an L-shaped prism, all counter-clockwise from outside;
and the edge cases: a dyadic heightfield solid, a box topped by a fan of needles, a box closed at a T-junction by a zero-area
triangle, a huge box beside a finely divided sphere, and a flat, two-sided plate."""
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


def _outward(v, f, normal):
    """f with every triangle whose normal points against its row of `normal` reversed"""
    v, f = np.asarray(v, np.float64), np.array(f)
    a, b, c = (v[f[:, k]] for k in range(3))
    flip = np.einsum("ij,ij->i", np.cross(b - a, c - a), normal) < 0
    f[flip] = f[flip][:, ::-1]
    return f


def grid_solid(xs, zs, top, y_bot):
    """The solid over the (x, z) grid xs x zs between a flat bottom at y_bot and the top vertices (xs[i], top[i, k], zs[k]), with
    vertical sides.  Top and bottom cells are split along the diagonal (i, k)-(i+1, k+1) when i + k is even and along the other
    diagonal when it is odd.  top == y_bot everywhere gives a flat, two-sided plate whose sides have zero area."""
    xs, zs, top = (np.asarray(a, np.float64) for a in (xs, zs, top))
    nx, nz = len(xs) - 1, len(zs) - 1
    X, Z = np.meshgrid(xs, zs, indexing="ij")
    bot = np.full_like(X, y_bot)
    v = np.concatenate([np.stack([X, top, Z], -1).reshape(-1, 3), np.stack([X, bot, Z], -1).reshape(-1, 3)])

    def T(i, k):
        return i * (nz + 1) + k

    def B(i, k):
        return (nx + 1) * (nz + 1) + i * (nz + 1) + k
    f, n = [], []
    for i in range(nx):
        for k in range(nz):
            if (i + k) % 2 == 0:
                halves = ([(i, k), (i + 1, k), (i + 1, k + 1)], [(i, k), (i + 1, k + 1), (i, k + 1)])
            else:
                halves = ([(i, k), (i + 1, k), (i, k + 1)], [(i + 1, k), (i + 1, k + 1), (i, k + 1)])
            for h in halves:
                f += [[T(*p) for p in h], [B(*p) for p in h]]
                n += [(0, 1, 0), (0, -1, 0)]
    for k in range(nz):
        for i, s in ((0, -1), (nx, 1)):
            f += [[T(i, k), T(i, k + 1), B(i, k + 1)], [T(i, k), B(i, k + 1), B(i, k)]]
            n += [(s, 0, 0)] * 2
    for i in range(nx):
        for k, s in ((0, -1), (nz, 1)):
            f += [[T(i, k), T(i + 1, k), B(i + 1, k)], [T(i, k), B(i + 1, k), B(i, k)]]
            n += [(0, 0, s)] * 2
    # orientation is topological: decide it on the solid lifted to a unit height, which also orients a flat plate's sides
    lifted = v.copy()
    lifted[:(nx + 1) * (nz + 1), 1] = y_bot + 1.0
    return v, _outward(lifted, f, np.asarray(n, np.float64))


def heightfield(n=16, seed=3, lo=(0.25, 0.25, 0.3125), step=2.0 ** -6):
    """A solid on an n x n grid of dyadic step in (x, z) with random dyadic heights in [lo.y + 1/4, lo.y + 1/4 + 15/256] over a flat
    bottom at lo.y: grid vertices, edge midpoints and cell centres are exact floats, so +y rays through them hit vertices, shared
    edges and (on the border) vertical faces exactly.  Returns (v, f, h) with h(x, z) the top surface in float64: the points
    inside are exactly those with x, z strictly inside the grid and lo.y < y < h(x, z).  Its slope is at most 15/4 per axis."""
    rng = np.random.default_rng(seed)
    xs, zs = lo[0] + step * np.arange(n + 1), lo[2] + step * np.arange(n + 1)
    top = lo[1] + 0.25 + rng.integers(0, 16, (n + 1, n + 1)) * 2.0 ** -8
    v, f = grid_solid(xs, zs, top, lo[1])

    def h(x, z):
        u, w = (np.asarray(x, np.float64) - xs[0]) / step, (np.asarray(z, np.float64) - zs[0]) / step
        i, k = np.clip(np.floor(u).astype(np.int64), 0, n - 1), np.clip(np.floor(w).astype(np.int64), 0, n - 1)
        u, w = u - i, w - k
        h00, h10, h01, h11 = top[i, k], top[i + 1, k], top[i, k + 1], top[i + 1, k + 1]
        even = np.where(u >= w, h00 + u * (h10 - h00) + w * (h11 - h10), h00 + w * (h01 - h00) + u * (h11 - h01))
        odd = np.where(u + w <= 1, h00 + u * (h10 - h00) + w * (h01 - h00), h11 + (1 - u) * (h01 - h11) + (1 - w) * (h10 - h11))
        return np.where((i + k) % 2 == 0, even, odd)
    return v, f, h


def needle_fan(lo=(0.3, 0.25, 0.3), hi=(0.5, 0.4, 0.5), widths=tuple(np.geomspace(2e-4, 2e-6, 25))):
    """A box whose top is a fan of needles from the corner (lo.x, hi.y, lo.z) to the edge x = hi.x, where their widths run from
    2e-4 down to 2e-6 (aspect ratios about 1e3 to 1e5) before four wide steps finish the edge.  The side x = hi.x is a fan of
    needles from its lower corner through the same edge vertices, so the mesh is closed without T-junctions."""
    z = lo[2] + np.concatenate([[0.0], np.cumsum(widths)])
    z = np.concatenate([z, np.linspace(z[-1], hi[2], 5)[1:]])
    K = len(z) - 1
    P = [(hi[0], hi[1], zk) for zk in z]
    A, C2 = (lo[0], hi[1], lo[2]), (lo[0], hi[1], hi[2])
    B0, B1, B2, B3 = (hi[0], lo[1], lo[2]), (hi[0], lo[1], hi[2]), (lo[0], lo[1], hi[2]), (lo[0], lo[1], lo[2])
    v = np.array(P + [A, C2, B0, B1, B2, B3], np.float64)
    a, c2, b0, b1, b2, b3 = range(K + 1, K + 7)
    f, n = [], []
    for k in range(K):
        f += [[a, k, k + 1], [b0, k, k + 1]]
        n += [(0, 1, 0), (1, 0, 0)]
    f += [[a, K, c2], [b0, K, b1]]
    n += [(0, 1, 0), (1, 0, 0)]
    for quad, nn in (((K, c2, b2, b1), (0, 0, 1)), ((c2, a, b3, b2), (-1, 0, 0)), ((a, 0, b0, b3), (0, 0, -1)),
                     ((b3, b0, b1, b2), (0, -1, 0))):
        p, q, r, s = quad
        f += [[p, q, r], [p, r, s]]
        n += [nn, nn]
    return v, _outward(v, f, np.asarray(n, np.float64))


def tjunction_box(lo=(0.3, 0.25, 0.3), hi=(0.5, 0.4, 0.45)):
    """A box whose top has a vertex M in the middle of its edge z = lo.z while the side z = lo.z uses that edge whole; the
    zero-area triangle (T0, M, T1) closes the junction."""
    T0, T1, T2, T3 = (lo[0], hi[1], lo[2]), (hi[0], hi[1], lo[2]), (hi[0], hi[1], hi[2]), (lo[0], hi[1], hi[2])
    B0, B1, B2, B3 = ((p[0], lo[1], p[2]) for p in (T0, T1, T2, T3))
    M = (0.5 * (lo[0] + hi[0]), hi[1], lo[2])
    v = np.array([T0, T1, T2, T3, B0, B1, B2, B3, M], np.float64)
    t0, t1, t2, t3, b0, b1, b2, b3, m = range(9)
    f = [[t0, m, t3], [m, t2, t3], [m, t1, t2]]
    n = [(0, 1, 0)] * 3
    for quad, nn in (((t0, t1, b1, b0), (0, 0, -1)), ((t1, t2, b2, b1), (1, 0, 0)), ((t2, t3, b3, b2), (0, 0, 1)),
                     ((t3, t0, b0, b3), (-1, 0, 0)), ((b0, b1, b2, b3), (0, -1, 0))):
        p, q, r, s = quad
        f += [[p, q, r], [p, r, s]]
        n += [nn, nn]
    f = _outward(v, f, np.asarray(n, np.float64))
    # the top uses M -> T0 and T1 -> M, the side T0 -> T1: the zero-area triangle takes each edge the other way
    return v, np.concatenate([f, [[t0, m, t1]]])


def box_and_sphere(subdiv, lo=(0.2, 0.2, 0.2), hi=(0.5, 0.4, 0.35), radius=0.03, center=(0.4, 0.3, 0.44)):
    """Two disjoint closed parts in one mesh: a box of 12 huge triangles and an icosphere of many tiny ones.  At subdiv 3 the mean
    triangle size is above 1/128 of the extent and sets the 3D cell; at subdiv 4 it is below, and the 128-cell cap binds."""
    vb, fb = box(lo, hi)
    vs, fs = icosphere(subdiv, radius, center)
    return np.concatenate([vb, vs]), np.concatenate([fb, fs + len(vb)])


def flat_plate(lo=(0.3, 0.3), hi=(0.5, 0.45), y=0.35, n=6):
    """A flat, two-sided n x n plate at height y, closed through zero-area sides: its bounding box has no extent in y."""
    return grid_solid(np.linspace(lo[0], hi[0], n + 1), np.linspace(lo[1], hi[1], n + 1), np.full((n + 1, n + 1), y), y)


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
    # a (nearly) zero-area triangle: va + vb + vc is rounding noise and the regions above are not to be trusted, but the triangle
    # is (within its tiny width) the union of its edges, so take the nearest of the three segments
    deg = ~(np.abs(den) > 1e-10 * (np.abs(va) + np.abs(vb) + np.abs(vc)))
    if np.any(deg):
        best, qs = None, None
        for s, e in ((a, b), (b, c), (c, a)):
            d = e - s
            dd = (d * d).sum(-1)
            with np.errstate(divide="ignore", invalid="ignore"):
                t = np.where(dd > 0, np.clip(((p - s) * d).sum(-1) / dd, 0.0, 1.0), 0.0)
            x = s + t[..., None] * d
            dist = ((p - x) ** 2).sum(-1)
            if best is None:
                best, qs = dist, x
            else:
                qs = np.where((dist < best)[..., None], x, qs)
                best = np.minimum(best, dist)
        q = np.where(deg[..., None], qs, q)
    return q


def distance(p, v, f, chunk=1024):
    p = np.asarray(p, np.float64)
    A, B, C = (np.asarray(v, np.float64)[np.asarray(f)[:, k]] for k in range(3))
    out = np.empty(len(p))
    for s in range(0, len(p), chunk):
        q = p[s:s + chunk, None, :]
        out[s:s + chunk] = np.sqrt(((_closest(q, A[None], B[None], C[None]) - q) ** 2).sum(-1).min(1))
    return out


def distance_within(p, v, f, reach):
    """distance() where it is at most reach, inf elsewhere: the same closest points over only the (point, triangle) pairs whose
    triangle's circumscribing ball about its centroid comes within reach of the point"""
    from scipy.spatial import cKDTree
    p, v, f = np.asarray(p, np.float64), np.asarray(v, np.float64), np.asarray(f)
    A, B, C = (v[f[:, k]] for k in range(3))
    cen = (A + B + C) / 3.0
    rad = np.max([np.linalg.norm(X - cen, axis=1) for X in (A, B, C)], axis=0)
    tree = cKDTree(p)
    out = np.full(len(p), np.inf)
    for s in range(0, len(f), 4096):
        near = tree.query_ball_point(cen[s:s + 4096], rad[s:s + 4096] + reach)
        ti = np.repeat(np.arange(s, s + len(near)), [len(x) for x in near])
        if len(ti) == 0:
            continue
        pi = np.concatenate([np.asarray(x, np.int64) for x in near])
        d = np.sqrt(((_closest(p[pi], A[ti], B[ti], C[ti]) - p[pi]) ** 2).sum(-1))
        np.minimum.at(out, pi, d)
    out[out > reach] = np.inf
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


def fill_ranges(v, origin, spacing):
    """sphk_mesh_fill's inclusive index ranges ((j0, j1), (i0, i1), (k0, k1)) along x, y, z over the float32 bounding box of v,
    with one index of margin on each side, computed in double as it does"""
    v = np.asarray(v, np.float32)
    lo, hi = v.min(0).astype(np.float64), v.max(0).astype(np.float64)
    o, s = np.float32(origin).astype(np.float64), float(np.float32(spacing))
    return tuple((int(np.floor((lo[a] - o[a]) / s)) - 1, int(np.floor((hi[a] - o[a]) / s)) + 1) for a in range(3))


def lattice(origin, spacing, ranges):
    """The points k_fill_flag forms, float32(o + float32(s * idx)) per axis, in lattice_point's order (y index outermost, then x,
    z innermost) over ranges = ((j0, j1), (i0, i1), (k0, k1))"""
    o, s = np.float32(origin), np.float32(spacing)
    (j0, j1), (i0, i1), (k0, k1) = ranges
    i, j, k = np.meshgrid(np.arange(i0, i1 + 1), np.arange(j0, j1 + 1), np.arange(k0, k1 + 1), indexing="ij")
    pos = np.empty(i.shape + (3,), np.float32)
    pos[..., 0] = o[0] + s * j.astype(np.float32)
    pos[..., 1] = o[1] + s * i.astype(np.float32)
    pos[..., 2] = o[2] + s * k.astype(np.float32)
    return pos.reshape(-1, 3)


def sphere_gap(p, radius, center):
    """signed distance to the ideal sphere (negative inside)"""
    return np.linalg.norm(np.asarray(p, np.float64) - center, axis=-1) - radius


def torus_gap(p, R, r, center):
    """signed distance to the ideal torus about the y axis (negative inside)"""
    d = np.asarray(p, np.float64) - center
    return np.hypot(np.hypot(d[..., 0], d[..., 2]) - R, d[..., 1]) - r


def _longest_edge(v, f):
    v = np.asarray(v, np.float64)
    a, b, c = (v[np.asarray(f)[:, k]] for k in range(3))
    return max(np.linalg.norm(b - a, axis=1).max(), np.linalg.norm(c - b, axis=1).max(), np.linalg.norm(a - c, axis=1).max())


# The gap g is 1-Lipschitz.  On a triangle with longest edge l, g differs from its linear interpolation of the vertex values by at
# most 1/2 M l^2, M bounding the spectral norm of g's Hessian within l of the vertices (its eigenvalues are the principal
# curvatures of the level surfaces).  So |g| <= band on the whole mesh, where band = max |g(vertex)| + 1/2 M l^2.  Then a point
# with g < -band is inside the mesh, one with g > band outside, and its distance to the mesh lies in [|g| - band, |g| + band].
def sphere_band(v, f, radius, center):
    g, l = float(np.abs(sphere_gap(v, radius, center)).max()), _longest_edge(v, f)
    return g + 0.5 * l * l / (radius - l - g)


def torus_band(v, f, R, r, center):
    g, l = float(np.abs(torus_gap(v, R, r, center)).max()), _longest_edge(v, f)
    return g + 0.5 * l * l * max(1.0 / (r - l - g), 1.0 / (R - r - l - g))


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
