"""Scenes from triangle meshes without a device (DESIGN.md section 2.12): the OBJ reader, sphk_mesh_properties against the float64
reference and analytic values, the exports, the refusals of the C-ABI, and the headless app's refusals (all before any CUDA call)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mesh_ref as R
from util import ROOT

CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")


def _meshes(pkg):
    from cpp_fluid_particles_b200 import meshes
    return meshes


def _mesh(meshes, vf):
    v, f = vf
    return meshes.Mesh(np.asarray(v, np.float32), f)


# ---- OBJ reader ------------------------------------------------------------------------------------------------------------------
def test_obj_quads_ngons_negative_indices_and_comments(pkg, built, tmp_path):
    meshes = _meshes(pkg)
    p = tmp_path / "a.obj"
    p.write_text("# a unit square and a pentagon\n"
                 "o thing\nvn 0 0 1\nvt 0 0\n"
                 "v 0 0 0\nv 1 0 0\nv 1 1 0 1.0\nv 0 1 0   # trailing comment\n"
                 "f 1/1/1 2/1/1 3/1/1 4/1/1\n"
                 "v 2 0 0\nv 3 0 0\nv 3 1 0\nv 2.5 2 0\nv 2 1 0\n"
                 "f -5//1 -4//1 -3//1 -2//1 -1//1\n"
                 "usemtl x\ns off\nl 1 2\n")
    m = meshes.load_obj(str(p))
    assert m.vertices.shape == (9, 3) and m.vertices.dtype == np.float32
    assert m.triangles.tolist() == [[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7], [4, 7, 8]]
    t = meshes.load_obj(str(p), 2.0, (0.5, 0.0, -1.0))
    assert np.array_equal(t.vertices, meshes.transform(m.vertices, 2.0, (0.5, 0.0, -1.0)))
    assert np.array_equal(t.vertices, np.float32(2.0) * m.vertices + np.float32([0.5, 0.0, -1.0]))


@pytest.mark.parametrize("text,line", [("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n", 4), ("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 0\n", 4),
                                       ("v 0 0 0\nv 1 x 0\nv 0 1 0\nf 1 2 3\n", 2), ("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 -4 3\n", 4),
                                       ("v 0 0 0\nv 1 0 0\nv 0 1 0\n\nf 1 2\n", 5), ("v 0 0 0\nv 1 0 nan\nv 0 1 0\nf 1 2 3\n", 2)])
def test_obj_errors_name_the_line(pkg, built, tmp_path, text, line):
    meshes = _meshes(pkg)
    p = tmp_path / "bad.obj"
    p.write_text(text)
    with pytest.raises(ValueError, match=f"bad.obj:{line}:"):
        meshes.load_obj(str(p))


# ---- mass properties -----------------------------------------------------------------------------------------------------------
def test_box_exact(pkg, built):
    meshes = _meshes(pkg)
    p = _mesh(meshes, R.box((0.25, 0.5, 0.125), (1.25, 2.5, 3.125))).properties()
    a, b, c = 1.0, 2.0, 3.0
    assert p["closed"] and p["volume"] == pytest.approx(6.0, rel=1e-15) and p["area"] == pytest.approx(22.0, rel=1e-15)
    assert np.allclose(p["centroid"], [0.75, 1.5, 1.625], rtol=1e-15, atol=0)
    V = 6.0
    I = [V * (b * b + c * c) / 12, V * (a * a + c * c) / 12, V * (a * a + b * b) / 12]
    assert np.allclose(p["inertia"][:3], I, rtol=1e-14) and np.all(np.abs(p["inertia"][3:]) < 1e-14)
    assert np.allclose(p["principal"], sorted(I), rtol=1e-14)


def _quat_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def test_rotated_box_recovers_moments_and_axes(pkg, built):
    meshes = _meshes(pkg)
    q = np.array([0.3, -0.5, 0.2, 0.8])
    q /= np.linalg.norm(q)
    Rq = _quat_matrix(q)
    ext = np.array([0.3, 0.1, 0.2])                                     # body x, y, z extents
    v, f = R.box(-ext / 2, ext / 2)
    v = v @ Rq.T + np.array([0.5, 0.4, 0.6])
    p = _mesh(meshes, (v, f)).properties()
    V = ext.prod()
    I = V * np.array([ext[1] ** 2 + ext[2] ** 2, ext[0] ** 2 + ext[2] ** 2, ext[0] ** 2 + ext[1] ** 2]) / 12
    order = np.argsort(I)
    assert np.allclose(p["principal"], I[order], rtol=1e-5)
    Rp = _quat_matrix(p["orientation"])
    assert np.linalg.det(Rp) == pytest.approx(1.0, abs=1e-12) and p["orientation"][3] >= 0
    for k in range(3):                                                   # principal axis k is the box's axis order[k], up to sign
        assert abs(abs(Rp[:, k] @ Rq[:, order[k]]) - 1.0) < 1e-5
    assert np.allclose(p["centroid"], [0.5, 0.4, 0.6], atol=1e-6)


@pytest.mark.parametrize("name", ["icosphere", "torus", "l_prism"])
def test_curved_meshes_against_reference(pkg, built, name):
    meshes = _meshes(pkg)
    vf = {"icosphere": lambda: R.icosphere(3, 0.12, (0.5, 0.4, 0.5)), "torus": lambda: R.torus(0.15, 0.05, 48, 24, (0.5, 0.3, 0.5)),
          "l_prism": lambda: R.l_prism((0.3, 0.2, 0.4), 0.1, 0.15)}[name]()
    m = _mesh(meshes, vf)
    p = m.properties()
    V, c, I = R.mass_properties(m.vertices, m.triangles)                # the float32 vertices the library saw
    assert p["closed"]
    assert abs(p["volume"] - V) <= 1e-12 * V
    assert np.max(np.abs(p["centroid"] - c)) <= 1e-12 * np.max(np.abs(c))
    ref = [I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]]
    assert np.max(np.abs(p["inertia"] - ref)) <= 1e-12 * np.max(np.abs(I))
    ev = np.linalg.eigvalsh(I)
    assert np.max(np.abs(p["principal"] - ev)) <= 1e-12 * ev.max()
    assert p["area"] == pytest.approx(R.area(m.vertices, m.triangles), rel=1e-12)
    # the principal axes diagonalise the tensor
    Rp = _quat_matrix(p["orientation"])
    D = Rp.T @ I @ Rp
    assert np.max(np.abs(D - np.diag(p["principal"]))) <= 1e-9 * ev.max()


def test_reversed_winding_gives_the_same_outputs(pkg, built):
    meshes = _meshes(pkg)
    v, f = R.torus(0.15, 0.05, 32, 16, (0.5, 0.3, 0.5))
    a = _mesh(meshes, (v, f)).properties()
    b = _mesh(meshes, (v, f[:, ::-1])).properties()
    assert a["closed"] and b["closed"]
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def test_open_plate_reports_area_only(pkg, built):
    meshes = _meshes(pkg)
    v, f = R.plate((0.2, 0.2), (0.6, 0.5), 0.3)
    p = _mesh(meshes, (v, f)).properties()
    assert not p["closed"] and p["area"] == pytest.approx(0.4 * 0.3, rel=1e-6)
    assert p["volume"] == 0.0 and not np.any(p["inertia"])
    v, f = R.box((0, 0, 0), (1, 1, 1))
    assert not _mesh(meshes, (v, f[:-1])).properties()["closed"]          # one triangle missing


def test_mesh_cube_matches_the_float_cube_formula(pkg, built):
    """a cube of side n sb as a mesh gives sph_headless --float's mass and moments (floating_cube)"""
    meshes = _meshes(pkg)
    sb = np.float32(0.99) * np.float32(1.0) / np.float32(2 * 50 - 1)
    n = int(round(0.1 / float(sb))) + 1
    side = np.float32(n) * sb
    rel = np.float32(0.6)
    fmpv = np.float32(76.596750762082e-6) / (np.float32(0.02) * np.float32(0.02) * np.float32(0.02))
    mass = rel * fmpv * side * side * side
    I = mass * side * side / np.float32(6.0)
    p = _mesh(meshes, R.box((0.4, 0.4, 0.4), (0.4 + float(side),) * 3)).properties()
    rho = float(rel) * float(fmpv)
    assert rho * p["volume"] == pytest.approx(float(mass), rel=1e-6)
    assert np.allclose(np.asarray(p["principal"]) * rho, float(I), rtol=1e-5)


def _bin_sides(v, f):
    """sphk_mesh_create's 3D cell side candidates: the mean bounding-box side of a triangle and 1/128 of the largest extent"""
    v = np.asarray(v, np.float32).astype(np.float64)
    t = v[np.asarray(f)]
    side = ((t.max(1) - t.min(1)).sum(1) / 3.0).mean()
    return side, (v.max(0) - v.min(0)).max() / 128.0


def test_edge_case_reference_meshes(pkg, built):
    """the meshes of test_gpu_mesh_edges.py: closed by the library's edge criterion, with the volumes their construction gives,
    a heightfield whose closed-form top matches its vertices, bins in the regime each mesh is meant for, and lattice() equal to
    scene.fluid_lattice bit for bit"""
    meshes = _meshes(pkg)
    v, f, h = R.heightfield()
    m = _mesh(meshes, (v, f))
    assert np.array_equal(m.vertices.astype(np.float64), v)                  # dyadic: exact in float32
    assert np.array_equal(h(v[:, 0], v[:, 2])[:len(v) // 2], v[:len(v) // 2, 1])
    tri = v[f]
    top = np.all(tri[:, :, 1] > 0.25, axis=1)                                # the top's prisms down to y = 0.25, exactly
    xz = np.cross(tri[top, 1] - tri[top, 0], tri[top, 2] - tri[top, 0])[:, 1]
    vol = (0.5 * xz * (tri[top, :, 1].mean(1) - 0.25)).sum()
    p = m.properties()
    assert p["closed"] and p["volume"] == pytest.approx(vol, rel=1e-12) and R.mass_properties(v, f)[0] == pytest.approx(vol, rel=1e-12)
    for vf, vol in ((R.needle_fan(), 0.2 * 0.15 * 0.2), (R.tjunction_box(), 0.2 * 0.15 * 0.15)):
        m = _mesh(meshes, vf)
        p = m.properties()
        assert p["closed"] and p["volume"] == pytest.approx(vol, rel=1e-6)
        assert R.mass_properties(m.vertices, m.triangles)[0] == pytest.approx(p["volume"], rel=1e-12)
    v, f = R.needle_fan()
    a, b, c = (v[f[:, k]] for k in range(3))
    edge = np.maximum(np.linalg.norm(b - a, axis=1), np.maximum(np.linalg.norm(c - b, axis=1), np.linalg.norm(a - c, axis=1)))
    aspect = edge ** 2 / np.linalg.norm(np.cross(b - a, c - a), axis=1)     # longest edge over the height onto it
    assert aspect.min() < 10 and 5e2 < np.sort(aspect)[-50] and aspect.max() > 1e5
    v, f = R.tjunction_box()
    a, b, c = (v[f[:, k]] for k in range(3))
    assert np.count_nonzero(np.linalg.norm(np.cross(b - a, c - a), axis=1) == 0) == 1
    for subdiv in (3, 4):
        vf = R.box_and_sphere(subdiv)
        m = _mesh(meshes, vf)
        p = m.properties()
        V = R.mass_properties(m.vertices, m.triangles)[0]
        vs, fs = R.icosphere(subdiv, 0.03, (0.4, 0.3, 0.44))
        band = R.sphere_band(vs, fs, 0.03, np.array([0.4, 0.3, 0.44])) * R.area(vs, fs)
        assert p["closed"] and p["volume"] == pytest.approx(V, rel=1e-12)
        assert abs(V - (0.3 * 0.2 * 0.15 + 4 / 3 * np.pi * 0.03 ** 3)) <= band
        side, cap = _bin_sides(*vf)
        assert side > cap if subdiv == 3 else side < cap          # the mean triangle sets the cell / the 128-cell cap binds
    # the flat plate: closed, a zero y extent, and no volume (properties refuses it, but still reports closed)
    v, f = R.flat_plate()
    pm = _mesh(meshes, (v, f))
    from cpp_fluid_particles_b200 import capi
    out, fl = np.zeros(18), C.c_int(0)
    P = lambda a: a.ctypes.data_as(C.c_void_p)           # noqa: E731
    assert capi.sphk().sphk_mesh_properties(P(pm.vertices), len(v), P(pm.triangles), len(f), P(out), C.byref(fl)) == -1
    assert fl.value & meshes.CLOSED and np.ptp(pm.vertices[:, 1]) == 0.0
    # the large curved meshes: closed, and the polyhedral volume within band x area of the ideal solid's
    for vf, ideal, band in (
            (R.icosphere(5, 0.3, (0.5, 0.45, 0.5)), 4 / 3 * np.pi * 0.3 ** 3,
             lambda v, f: R.sphere_band(v, f, 0.3, np.array([0.5, 0.45, 0.5]))),
            (R.torus(0.25, 0.08, 256, 128, (0.5, 0.45, 0.5)), 2 * np.pi ** 2 * 0.25 * 0.08 ** 2,
             lambda v, f: R.torus_band(v, f, 0.25, 0.08, np.array([0.5, 0.45, 0.5])))):
        m = _mesh(meshes, vf)
        p = m.properties()
        vv = m.vertices.astype(np.float64)
        V = R.mass_properties(vv, m.triangles)[0]
        assert p["closed"] and p["volume"] == pytest.approx(V, rel=1e-12)
        assert abs(V - ideal) <= band(vv, m.triangles) * R.area(vv, m.triangles)
    # lattice() is scene.fluid_lattice over its own ranges, and fill_ranges() is the box fill's
    o, s = (0.135, 0.055, 0.135), float(pkg.scene.SPACING)
    assert np.array_equal(R.lattice(o, s, ((0, 9), (0, 13), (0, 9))).view(np.uint32), pkg.scene.fluid_lattice(10, 14, 10, o).view(np.uint32))
    lo = np.array(o) - s / 2
    hi = np.array(o) + s * np.array([9, 13, 9]) + s / 2
    v, _ = R.box(lo, hi)
    pts = R.lattice(o, s, R.fill_ranges(v, o, s))
    v32 = np.float32(v)
    inside = np.all((pts > v32.min(0)) & (pts < v32.max(0)), axis=1)
    assert np.array_equal(pts[inside].view(np.uint32), pkg.scene.fluid_lattice(10, 14, 10, o).view(np.uint32))


# ---- exports and refusals ------------------------------------------------------------------------------------------------------
def test_exports(pkg, built):
    from cpp_fluid_particles_b200 import capi
    L, A = capi.sphk(), capi.app_lib()
    for name in ("sphk_mesh_transform", "sphk_mesh_properties", "sphk_mesh_create", "sphk_mesh_destroy", "sphk_mesh_classify",
                 "sphk_mesh_fill", "sphk_mesh_sample_surface"):
        assert hasattr(L, name) and name in capi.SPHK_FUNCTIONS
    for name in ("sph_app_load_obj", "sph_app_load_obj_error"):
        assert hasattr(A, name) and name in capi.SPH_APP_FUNCTIONS


def test_refusals_without_a_device(pkg, built):
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    v = np.zeros((3, 3), np.float32)
    v[1, 0] = v[2, 1] = 1.0
    f = np.array([[0, 1, 2]], np.int32)
    out = np.zeros(18)
    fl = C.c_int(0)
    P = lambda a: a.ctypes.data_as(C.c_void_p)           # noqa: E731
    t = (C.c_float * 3)(0, 0, 0)
    assert L.sphk_mesh_transform(None, 3, C.c_float(1), t, P(v)) == -1
    assert L.sphk_mesh_transform(P(v), 3, C.c_float(1), t, P(v)) == -1                      # aliased
    assert L.sphk_mesh_transform(P(v), 3, C.c_float(float("nan")), t, P(np.empty_like(v))) == -1
    assert L.sphk_mesh_properties(P(v), 3, P(f), 1, None, C.byref(fl)) == -1
    assert L.sphk_mesh_properties(P(v), 3, P(np.array([[0, 1, 3]], np.int32)), 1, P(out), C.byref(fl)) == -1
    bad = v.copy(); bad[0, 0] = np.inf
    assert L.sphk_mesh_properties(P(bad), 3, P(f), 1, P(out), C.byref(fl)) == -1
    assert L.sphk_mesh_properties(P(v), 3, P(f), 0, P(out), C.byref(fl)) == -1
    h = C.c_void_p(123)
    assert L.sphk_mesh_create(C.byref(h), P(v), 3, P(np.array([[0, 1, -1]], np.int32)), 1, None) == -1 and not h.value
    assert L.sphk_mesh_create(None, P(v), 3, P(f), 1, None) == -1
    n = C.c_int(0)
    assert L.sphk_mesh_classify(None, P(v), 1, C.c_float(0), P(f)) == -1
    assert L.sphk_mesh_fill(None, C.c_float(0.02), t, C.c_float(0), P(v), 1, C.byref(n)) == -1
    assert L.sphk_mesh_sample_surface(None, C.c_float(0.02), P(v), 1, C.byref(n)) == -1
    L.sphk_mesh_destroy(None)


def _obj(tmp_path, name, vf):
    return R.write_obj(tmp_path / name, *vf)


@pytest.mark.parametrize("case", ["ranks", "open_body", "open_fluid", "open_obstacle", "outside", "parse", "stir", "spec"])
def test_headless_refusals(pkg, built, tmp_path, case):
    """refused before any CUDA call (exit code 2), with a message that names the option"""
    torus = _obj(tmp_path, "torus.obj", R.torus(0.12, 0.04, 24, 12, (0.5, 0.3, 0.5)))
    plate = _obj(tmp_path, "plate.obj", R.plate((0.3, 0.3), (0.6, 0.6), 0.4))
    big = _obj(tmp_path, "big.obj", R.box((0.1, 0.1, 0.1), (0.5, 0.5, 1.2)))
    bad = tmp_path / "bad.obj"
    bad.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 9\n")
    args, opt = {"ranks": (["--obstacle", torus, "--ranks", "2"], "--obstacle"),
                 "open_body": (["--mesh-body", plate + ",0.5"], "--mesh-body"),
                 "open_fluid": (["--fluid-mesh", plate], "--fluid-mesh"),
                 "open_obstacle": (["--obstacle", plate], "--obstacle"),
                 "outside": (["--obstacle", big], "--obstacle"),
                 "parse": (["--obstacle", str(bad)], "--obstacle"),
                 "stir": (["--mesh-body", torus + ",1", "--stir", "2"], "--mesh-body"),
                 "spec": (["--mesh-body", torus + ",1,2"], "--mesh-body")}[case]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([CLI, "--quiet", "--frames", "1"] + args, capture_output=True, text=True, timeout=60, env=env)
    assert r.returncode == 2, (r.returncode, r.stderr)
    assert opt in r.stderr, r.stderr
    if case == "parse":
        assert "bad.obj:4:" in r.stderr
