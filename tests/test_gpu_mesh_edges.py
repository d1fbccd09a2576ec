"""The mesh scene builders on the GPU (DESIGN.md section 2.12) where they can break, against float64 and closed forms (mesh_ref.py):
exact +y ray ties on a dyadic heightfield and through the vertices of large meshes, distances to needle and zero-area triangles,
bins whose cell the mean triangle or the 128-cell cap sets, a flat bounding box, fills of more than 2M points compared point for
point in lattice order, Poisson-disk sampling at 1000 cells per axis and far from the origin, and the capacity contract of fill
and sample through the C-ABI.  The only allowance is a 1e-6 band about the surface (or about the clearance, for the near bit);
on the large meshes that band is widened by the facets' proven distance from the ideal sphere or torus."""
import ctypes as C
import functools

import numpy as np
import pytest

import mesh_ref as R
from util import bits

pytestmark = pytest.mark.gpu

BAND = 1e-6


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _mesh(v, f):
    from cpp_fluid_particles_b200 import meshes
    return meshes.Mesh(np.asarray(v, np.float32), f)


C_ICO = np.array([0.5, 0.45, 0.5])


@functools.lru_cache(maxsize=None)
def _large(name):
    """(v, f, gap, band) of the large curved meshes: gap is the signed distance to the ideal surface, and the mesh lies within band
    of it (mesh_ref.sphere_band / torus_band, on the float32 vertices)"""
    if name == "icosphere":
        v, f = R.icosphere(7, 0.3, C_ICO)                       # 327,680 triangles
        v = np.float32(v).astype(np.float64)
        return v, f, (lambda p: R.sphere_gap(p, 0.3, C_ICO)), R.sphere_band(v, f, 0.3, C_ICO)
    v, f = R.torus(0.25, 0.08, 512, 256, C_ICO)                  # 262,144 triangles
    v = np.float32(v).astype(np.float64)
    return v, f, (lambda p: R.torus_gap(p, 0.25, 0.08, C_ICO)), R.torus_band(v, f, 0.25, 0.08, C_ICO)


def _near_known(g, band, c):
    """(known, near) from the gap: the distance to the mesh lies in [|g| - band, |g| + band]"""
    a = np.abs(g)
    near = a + band <= c - BAND
    return near | (a - band > c + BAND), near


def _check_classify(m, p, inside, inside_known, c, near, near_known):
    fl = m.classify(p, c)
    assert np.array_equal((fl[inside_known] & 1) == 1, inside[inside_known]), \
        np.flatnonzero(((fl & 1) == 1) != inside)[:10]
    assert np.array_equal((fl[near_known] & 2) == 2, near[near_known]), np.flatnonzero(((fl & 2) == 2) != near)[:10]


# ---- classify ---------------------------------------------------------------------------------------------------------------------
def test_heightfield_exact_ray_ties(pkg, built):
    """every vertex, edge midpoint, cell centre and quarter point of the dyadic heightfield, below, inside and above it: the inside
    bit is the closed form lo.y < y < h(x, z) for every point, with no band (all points are 2^-9 / sqrt(1 + 2 (15/4)^2) > 3e-4 from
    the surface by construction).  On the border the rays run inside the vertical faces; only points outside the solid go there."""
    _gpu()
    v, f, h = R.heightfield()
    m = _mesh(v, f)
    q = 2.0 ** -8                                               # a quarter of the grid step
    xs, zs = 0.25 + q * np.arange(65), 0.3125 + q * np.arange(65)
    X, Z = (a.ravel() for a in np.meshgrid(xs, zs, indexing="ij"))
    H = h(X, Z)
    border = (X == xs[0]) | (X == xs[-1]) | (Z == zs[0]) | (Z == zs[-1])
    levels = (0.25 - 2.0 ** -7 + 0 * H, 0.25 + 2.0 ** -8 + 0 * H, H - 2.0 ** -9, H + 2.0 ** -9, H + 2.0 ** -5)
    p = np.concatenate([np.stack([X, y, Z], 1)[~border if k in (1, 2) else slice(None)] for k, y in enumerate(levels)])
    assert np.array_equal(np.float32(p).astype(np.float64), p)             # every query point is exact in float32
    x, y, z = p.T
    inside = (x > xs[0]) & (x < xs[-1]) & (z > zs[0]) & (z < zs[-1]) & (y > 0.25) & (y < h(x, z))
    fl = m.classify(p, 0.0)
    assert np.array_equal((fl & 1) == 1, inside), np.flatnonzero(((fl & 1) == 1) != inside)[:10]
    assert np.count_nonzero(inside) == 2 * 63 * 63
    # outside the (x, z) bounding box, some just outside it: clamped into the edge columns, still outside
    rng = np.random.default_rng(11)
    far = rng.uniform((0.0, 0.2, 0.0), (0.8, 0.6, 0.9), (20000, 3))
    far = far[(far[:, 0] < xs[0]) | (far[:, 0] > xs[-1]) | (far[:, 2] < zs[0]) | (far[:, 2] > zs[-1])]
    edge = rng.uniform((0.25, 0.2, 0.3125), (0.5, 0.6, 0.5625), (4000, 3))
    edge[:1000, 0], edge[1000:2000, 0] = xs[0] - 2.0 ** -12, xs[-1] + 2.0 ** -12
    edge[2000:3000, 2], edge[3000:, 2] = zs[0] - 2.0 ** -12, zs[-1] + 2.0 ** -12
    assert np.all(m.classify(np.concatenate([far, edge]), 0.0) & 1 == 0)


@pytest.mark.parametrize("name", ["icosphere", "torus"])
def test_large_mesh_vertex_rays_and_2m_points(pkg, built, name):
    """rays through every vertex's (x, z) -- fans of 5 and 6 triangles, and on the torus silhouette vertices where the ray grazes
    -- at nine heights, and 2M seeded points in the bounding box: inside and near bits against the ideal surface"""
    _gpu()
    v, f, gap, band = _large(name)
    m = _mesh(v, f)
    lo, hi = v.min(0), v.max(0)
    c = 0.004
    levels = [lo[1] - 0.01, lo[1] + 0.05, C_ICO[1] - 0.03, C_ICO[1], C_ICO[1] + 0.03, hi[1] - 0.05, hi[1] + 0.01]
    ys = np.concatenate([np.full(len(v), y) for y in levels] + [v[:, 1] - 0.003, v[:, 1] + 0.003])
    p = np.float32(np.stack([np.tile(v[:, 0], len(levels) + 2), ys, np.tile(v[:, 2], len(levels) + 2)], 1))
    rng = np.random.default_rng(5)
    p = np.concatenate([p, np.float32(lo - 0.01 + rng.random((2_000_000, 3)) * (hi - lo + 0.02))])
    gp = gap(p.astype(np.float64))
    known, near = _near_known(gp, band, c)
    inside_known = np.abs(gp) > band + BAND
    _check_classify(m, p, gp < 0, inside_known, c, near, known)
    assert np.count_nonzero(inside_known) > 0.98 * len(p) and np.count_nonzero(known) > 0.98 * len(p)
    if name == "torus":                                          # the silhouette (w = 0, pi) vertices' rays were checked
        sil = np.abs(v[:, 1] - C_ICO[1]) < 1e-7
        assert np.count_nonzero(sil) == 2 * 512 and np.all(inside_known[:len(v)][sil])


def _sliver_points(v, seed, n=8000):
    """seeded points around the mesh, half of them within 0.02 of its top face"""
    rng = np.random.default_rng(seed)
    lo, hi = v.min(0), v.max(0)
    a = lo - 0.02 + rng.random((n, 3)) * (hi - lo + 0.04)
    a[::2, 1] = hi[1] + rng.uniform(-0.02, 0.02, len(a[::2]))
    return np.float32(a)


@pytest.mark.parametrize("name", ["needle_fan", "tjunction_box", "box_and_sphere_3", "box_and_sphere_4", "flat_plate"])
def test_near_and_inside_on_edge_meshes(pkg, built, name):
    """needles of aspect 1e3-1e5, a zero-area T-junction triangle, bins set by the mean triangle and by the 128-cell cap, a flat
    bounding box: the near bit at four clearances equals the float64 distance test outside a 1e-6 band about the clearance,
    and the inside bit the float64 winding number for every point farther than 1e-6 from the surface"""
    _gpu()
    vf = {"needle_fan": R.needle_fan, "tjunction_box": R.tjunction_box, "box_and_sphere_3": lambda: R.box_and_sphere(3),
          "box_and_sphere_4": lambda: R.box_and_sphere(4), "flat_plate": R.flat_plate}[name]()
    m = _mesh(*vf)
    v = m.vertices.astype(np.float64)
    p = _sliver_points(v, 13)
    if name == "needle_fan":                                     # over and under the needles, near their apex and along them
        rng = np.random.default_rng(17)
        q = np.stack([rng.uniform(0.29, 0.51, 8000), 0.4 + rng.uniform(-0.012, 0.012, 8000), rng.uniform(0.2995, 0.3012, 8000)], 1)
        p = np.concatenate([p, np.float32(q)])
    elif name == "tjunction_box":                                # around the edge the zero-area triangle lies on
        rng = np.random.default_rng(19)
        q = np.stack([rng.uniform(0.28, 0.52, 8000), 0.4 + rng.uniform(-0.012, 0.012, 8000), 0.3 + rng.uniform(-0.012, 0.012, 8000)], 1)
        p = np.concatenate([p, np.float32(q)])
    elif name.startswith("box_and_sphere"):                      # around the finely divided sphere
        rng = np.random.default_rng(23)
        d = rng.normal(size=(8000, 3))
        q = np.array([0.4, 0.3, 0.44]) + d / np.linalg.norm(d, axis=1)[:, None] * rng.uniform(0.0, 0.045, (8000, 1))
        p = np.concatenate([p, np.float32(q)])
    d = R.distance_within(p, v, m.triangles, 0.02)               # inf beyond: farther than every clearance
    if name.startswith("box_and_sphere"):                        # two closed parts: the sphere's winding is 0 outside its box
        fb, fs = m.triangles[:12], m.triangles[12:]
        w = R.winding_number(p, v, fb)
        vs = v[fs.ravel()]
        ins = np.all((p >= vs.min(0)) & (p <= vs.max(0)), axis=1)
        w[ins] += R.winding_number(p[ins], v, fs, chunk=256)
    else:
        w = R.winding_number(p, v, m.triangles, chunk=256)
    if name == "flat_plate":
        assert np.all(np.abs(w) < 1e-9)                          # no inside at all
    inside_known = d > BAND
    fl0 = m.classify(p, 0.0)
    assert np.array_equal((fl0[inside_known] & 1) == 1, w[inside_known] > 0.5)
    for c in (0.0005, 0.002, 0.006, 0.015):
        known = np.abs(d - c) > BAND
        fl = m.classify(p, c)
        bad = np.flatnonzero(known & (((fl & 2) == 2) != (d <= c)))
        assert len(bad) == 0, (c, len(bad), p[bad[:5]], d[bad[:5]], fl[bad[:5]])
        assert np.array_equal(fl & 1, fl0 & 1)


# ---- fill ---------------------------------------------------------------------------------------------------------------------------
def _lattice_indices(out, origin, spacing, ranges):
    """the lattice index of each output point, checked bit for bit against mesh_ref.lattice's point"""
    (j0, j1), (i0, i1), (k0, k1) = ranges
    o, s = np.float32(origin).astype(np.float64), float(np.float32(spacing))
    jik = np.rint((out.astype(np.float64) - o) / s).astype(np.int64)
    idx = ((jik[:, 1] - i0) * (j1 - j0 + 1) + (jik[:, 0] - j0)) * (k1 - k0 + 1) + (jik[:, 2] - k0)
    return idx


def _check_fill(m, spacing, origin, clearance, keep, known):
    """the fill equals the reference lattice filtered by keep, in lattice order, for every point where known"""
    ranges = R.fill_ranges(m.vertices, origin, spacing)
    L = R.lattice(origin, spacing, ranges)
    assert len(keep) == len(L)
    out = m.fill(spacing, origin, clearance)
    idx = _lattice_indices(out, origin, spacing, ranges)
    assert np.all((idx >= 0) & (idx < len(L)))
    assert np.array_equal(bits(L[idx]), bits(out)), "a fill point is not a lattice point"
    assert np.all(np.diff(idx) > 0), "not in lattice order"
    got = np.zeros(len(L), bool)
    got[idx] = True
    bad = np.flatnonzero(known & (got != keep))
    assert len(bad) == 0, (len(bad), L[bad[:5]], keep[bad[:5]])
    return out


def test_fill_heightfield(pkg, built):
    """the heightfield's fill: inside by the closed form, clearance by the float64 distance (exact for every point that a lower
    bound does not already put far from the surface)"""
    _gpu()
    v, f, h = R.heightfield()
    m = _mesh(v, f)
    s, o, c = 0.0043, (0.0131, 0.0177, 0.0119), 0.005
    L = R.lattice(o, s, R.fill_ranges(m.vertices, o, s)).astype(np.float64)
    x, y, z = L.T
    inb = (x > 0.25) & (x < 0.5) & (z > 0.3125) & (z < 0.5625)
    hh = h(np.clip(x, 0.25, 0.5), np.clip(z, 0.3125, 0.5625))
    inside = inb & (y > 0.25) & (y < hh)
    cos = 1.0 / np.sqrt(1.0 + 2.0 * (15.0 / 4.0) ** 2)          # the steepest facet's normal against the vertical
    # lower bounds of the distance to the surface: inside, the gaps to the top (along the slope) and to the five planes; outside,
    # the gap to the bounding box and, over the grid, the gap above the top
    lower_in = np.minimum.reduce([(hh - y) * cos, y - 0.25, x - 0.25, 0.5 - x, z - 0.3125, 0.5625 - z])
    out = np.maximum.reduce([0.25 - x, x - 0.5, 0.25 - y, y - hh.max(), 0.3125 - z, z - 0.5625, np.zeros_like(x)])
    lower_out = np.maximum(out, np.where(inb, (y - hh) * cos, 0.0))
    exact = np.where(inside, lower_in <= c + 1e-3, lower_out <= 1e-5)
    d = np.where(inside, lower_in, lower_out)
    d[exact] = np.minimum(R.distance_within(L[exact], v, f, c + 2e-3), np.maximum(d[exact], c + 2e-3))
    known = (d > BAND) & (~inside | (np.abs(d - c) > BAND))
    _check_fill(m, s, o, c, inside & (d > c), known)


@pytest.mark.parametrize("name", ["icosphere", "torus"])
def test_fill_large_meshes(pkg, built, name):
    """the icosphere's fill makes more than 2M points (past every block boundary of the scan); both are equal to the lattice
    filtered by the ideal surface outside the band, and two calls give the same bits"""
    _gpu()
    v, f, gap, band = _large(name)
    m = _mesh(v, f)
    s, o, c = (0.0037, (0.0013, 0.0021, 0.0017), 0.0037) if name == "icosphere" else (0.0029, (0.0011, 0.0023, 0.0007), 0.002)
    L = R.lattice(o, s, R.fill_ranges(m.vertices, o, s))
    g = gap(L.astype(np.float64))
    keep = (g < 0) & (-g - band > c + BAND)                     # inside, and farther than c from the mesh
    drop = (g > band + BAND) | (np.abs(g) + band <= c - BAND)   # outside, or within c of the mesh
    out = _check_fill(m, s, o, c, keep, keep | drop)
    if name == "icosphere":
        assert len(out) >= 2_000_000
    assert np.array_equal(bits(out), bits(m.fill(s, o, c)))


# ---- sample -------------------------------------------------------------------------------------------------------------------------
def _check_sample(m, r, tri_subset=None):
    """minimum pairwise distance >= r (the kernel's own double test) and every point of a float64 r/8 sampling within
    r (1 + 1/(4 sqrt 3)) + delta of a sample: a candidate is within r/(4 sqrt 3) of every surface point near it and within r of a
    sample, and delta = 2^-20 max |coordinate| bounds the float rounding of the candidate's barycentric combination"""
    from scipy.spatial import cKDTree
    s = m.sample_surface(r).astype(np.float64)
    r = float(np.float32(r))
    tree = cKDTree(s)
    _, nn = tree.query(s, k=2)
    d2 = ((s - s[nn[:, 1]]) ** 2).sum(1)
    assert d2.min() >= r * r * (1 - 2.0 ** -50), np.sqrt(d2.min()) / r
    v = m.vertices.astype(np.float64)
    f = m.triangles if tri_subset is None else m.triangles[tri_subset]
    ref = R.surface_points(v, f, r / 8)
    d, _ = tree.query(ref)
    delta = 2.0 ** -20 * float(np.abs(v).max())
    assert d.max() <= r * (1 + 1 / (4 * np.sqrt(3))) + delta, d.max() / r
    return s


@pytest.mark.parametrize("name", ["needle_fan", "icosphere_1000_cells", "far_from_origin"])
def test_sample_edges(pkg, built, name):
    _gpu()
    if name == "needle_fan":
        m = _mesh(*R.needle_fan())
        _check_sample(m, 0.01)
    elif name == "icosphere_1000_cells":
        v, f = R.icosphere(6, 0.3, C_ICO)
        m = _mesh(v, f)
        r = float(np.ptp(m.vertices, axis=0).max()) / 1000.0
        subset = np.random.default_rng(3).choice(len(f), 600, replace=False)
        s = _check_sample(m, r, subset)
        assert len(s) > 1_000_000
    else:
        from cpp_fluid_particles_b200 import meshes
        v, f = R.icosphere(3, 0.1)
        m = meshes.Mesh(np.float32(v), f, 1.0, (64.0, 64.0, 64.0))
        _check_sample(m, 0.005)


# ---- capacity -----------------------------------------------------------------------------------------------------------------------
SENTINEL = 0x7FC0DEAD                                            # a NaN bit pattern neither call writes


def _raw(m, which, buf, cap, args):
    import torch
    from cpp_fluid_particles_b200 import capi
    n = C.c_int(-1)
    L = capi.sphk()
    if which == "fill":
        s, o, c = args
        rc = L.sphk_mesh_fill(m._mesh(), C.c_float(s), (C.c_float * 3)(*o), C.c_float(c), C.c_void_p(buf.data_ptr()), C.c_int(cap),
                              C.byref(n))
    else:
        rc = L.sphk_mesh_sample_surface(m._mesh(), C.c_float(args), C.c_void_p(buf.data_ptr()), C.c_int(cap), C.byref(n))
    torch.cuda.synchronize()
    return rc, n.value


@pytest.mark.parametrize("which", ["fill", "sample"])
def test_capacity(pkg, built, which):
    """through the C-ABI into a buffer whose sentinel tail is longer than the whole output: capacity == count writes the output
    and nothing past it; count - 1 and 0 report count and write nothing"""
    _gpu()
    import torch
    m = _mesh(*R.torus(0.1, 0.035, 48, 24, (0.45, 0.3, 0.4)))
    args = (0.006, (0.0, 0.0, 0.0), 0.0024) if which == "fill" else 0.0102
    big = torch.empty((100_000, 3), dtype=torch.int32, device="cuda")
    rc, count = _raw(m, which, big, len(big), args)
    assert rc == 0 and 500 < count < len(big)
    full = big[:count].cpu().numpy().view(np.float32)
    for cap in (count, count - 1, 0):
        buf = torch.full((2 * count + 64, 3), SENTINEL, dtype=torch.int32, device="cuda")
        rc, n = _raw(m, which, buf, cap, args)
        assert rc == 0 and n == count, (cap, rc, n)
        got = buf.cpu().numpy()
        if cap == count:
            assert np.array_equal(got[:count].view(np.uint32), bits(full))
            assert np.all(got[count:] == SENTINEL)
        else:
            assert np.all(got == SENTINEL), cap
