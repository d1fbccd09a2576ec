"""Scenes from triangle meshes on the GPU (DESIGN.md section 2.12): classify, fill and sample against the float64 reference
(mesh_ref.py), the layers against each other bit for bit, and the physics of mesh obstacles and bodies on all three solvers."""
import json
import os
import subprocess

import numpy as np
import pytest

import mesh_ref as R
from util import ROOT, bits

pytestmark = pytest.mark.gpu

CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
SOLVERS = ["wcsph", "dfsph", "pbd"]
SB = float(np.float32(0.99) * np.float32(0.5) / np.float32(2 * 13 - 1))     # the mini scene's boundary spacing (box 0.5, 13 cells)


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _m():
    from cpp_fluid_particles_b200 import meshes
    return meshes


CLOSED = {
    "cube": lambda: R.box((0.3, 0.2, 0.35), (0.5, 0.4, 0.55)),
    "icosphere": lambda: R.icosphere(3, 0.1, (0.4, 0.3, 0.45)),
    "torus": lambda: R.torus(0.1, 0.035, 48, 24, (0.45, 0.3, 0.4)),
    "l_prism": lambda: R.l_prism((0.3, 0.2, 0.3), 0.08, 0.1),
}


def _mesh(vf):
    return _m().Mesh(np.asarray(vf[0], np.float32), vf[1])


# ---- geometry -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CLOSED))
def test_classify_against_winding_number_and_distance(pkg, built, name):
    _gpu()
    m = _mesh(CLOSED[name]())
    lo, hi = m.vertices.min(0), m.vertices.max(0)
    rng = np.random.default_rng(7)
    p = (lo - 0.03 + rng.random((3000, 3)) * (hi - lo + 0.06)).astype(np.float32)
    c = 0.01
    fl = m.classify(p, c)
    w = R.winding_number(p, m.vertices, m.triangles)
    d = R.distance(p, m.vertices, m.triangles)
    far = d > 1e-5
    assert np.array_equal((fl[far] & 1) == 1, w[far] > 0.5)
    band = np.abs(d - c) > 1e-6
    assert np.array_equal(((fl & 2) == 2)[band], (d <= c)[band])
    assert 200 < np.count_nonzero(fl & 1) < 2800


def test_classify_rays_through_vertices_and_edges(pkg, built):
    """a lattice whose +y rays pass exactly through the cube's vertices and edges: the exact inside count"""
    _gpu()
    m = _mesh(R.box((0.25, 0.25, 0.25), (0.75, 0.75, 0.75)))
    g = np.arange(0, 1.0001, 0.125, dtype=np.float32)          # hits x, z = 0.25, 0.75 exactly; y = 0.25, 0.75 on faces
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    p = np.stack([x, y, z], -1).reshape(-1, 3)
    fl = m.classify(p, 0.0)
    strict = np.all((p > 0.25) & (p < 0.75), axis=1)
    on = np.all((p >= 0.25) & (p <= 0.75), axis=1) & ~strict
    assert np.array_equal((fl[~on] & 1) == 1, strict[~on])
    assert np.count_nonzero(fl[~on] & 1) == 27
    assert np.all(fl[on] & 2)


def test_fill_box_is_the_fluid_lattice(pkg, built):
    _gpu()
    nx, ny, nz = 10, 14, 10
    origin = (0.135, 0.055, 0.135)
    s = float(pkg.scene.SPACING)
    lo = np.array(origin) - s / 2
    hi = np.array(origin) + s * (np.array([nx, ny, nz]) - 1) + s / 2
    got = _mesh(R.box(lo, hi)).fill(s, origin, 0.0)
    ref = pkg.scene.fluid_lattice(nx, ny, nz, origin)
    assert got.shape == ref.shape and np.array_equal(bits(got), bits(ref))


@pytest.mark.parametrize("name", ["icosphere", "torus"])
def test_fill_curved(pkg, built, name):
    _gpu()
    vf = {"icosphere": lambda: R.icosphere(4, 0.15, (0.5, 0.4, 0.5)), "torus": lambda: R.torus(0.16, 0.06, 96, 48, (0.5, 0.4, 0.5))}[name]()
    m = _mesh(vf)
    s, c = 0.006, 0.0024            # the tube of the torus is 10 spacings across: the lattice count converges to V / s^3
    p = m.fill(s, (0.0, 0.0, 0.0), c)
    fl = m.classify(p, c)
    assert np.all(fl == 1)
    assert np.all(R.winding_number(p[::7], m.vertices, m.triangles) > 0.5)
    V = m.properties()["volume"]
    assert abs(len(m.fill(s, (0.0, 0.0, 0.0), 0.0)) - V / s ** 3) <= 0.02 * V / s ** 3


def _pairwise_min(p):
    from scipy.spatial import cKDTree
    d, _ = cKDTree(p.astype(np.float64)).query(p.astype(np.float64), k=2)
    return d[:, 1].min()


@pytest.mark.parametrize("name", ["plate", "cube", "icosphere", "torus", "l_prism"])
def test_sample_surface(pkg, built, name):
    _gpu()
    from scipy.spatial import cKDTree
    vf = R.plate((0.2, 0.3), (0.6, 0.5), 0.4) if name == "plate" else CLOSED[name]()
    m = _mesh(vf)
    r = 0.0102
    s = m.sample_surface(r)
    assert len(s) > 10
    ext = float(np.max(m.vertices.max(0) - m.vertices.min(0)))
    assert R.distance(s, m.vertices, m.triangles).max() <= 1e-6 * ext
    assert _pairwise_min(s) >= r * (1 - 1e-12)
    ref = R.surface_points(m.vertices, m.triangles, r / 8)
    d, _ = cKDTree(s.astype(np.float64)).query(ref)
    assert d.max() <= r + r / 4
    assert np.array_equal(bits(s), bits(m.sample_surface(r)))


# ---- layers -----------------------------------------------------------------------------------------------------------------------
def _mini(solver):
    return [CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135",
            "0.055", "0.135", "--quiet"] + (["--iters", "4"] if solver != "wcsph" else [])


def _run(args):
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_emit_scene_obstacle_matches_python(pkg, built, tmp_path):
    _gpu()
    meshes = _m()
    obj = R.write_obj(tmp_path / "torus.obj", *R.torus(0.08, 0.03, 32, 16))
    prefix = str(tmp_path / "scene")
    _run(_mini("dfsph") + ["--obstacle", obj + ",1,0.25,0.12,0.25", "--emit-scene", prefix])
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    m = meshes.load_obj(obj, 1.0, (0.25, 0.12, 0.25))
    boundary = np.concatenate([sc.boundary, m.sample_surface(SB)])
    flags = m.classify(sc.fluid, SB)
    fluid = sc.fluid[flags == 0]
    assert np.array_equal(bits(np.fromfile(prefix + ".boundary.f32", np.float32).reshape(-1, 3)), bits(boundary))
    assert np.array_equal(bits(np.fromfile(prefix + ".fluid.f32", np.float32).reshape(-1, 3)), bits(fluid))
    assert len(fluid) < len(sc.fluid)


def test_fluid_mesh_box_is_the_block_run(pkg, built, tmp_path):
    _gpu()
    s = float(pkg.scene.SPACING)
    o = np.array([0.135, 0.055, 0.135])
    obj = R.write_obj(tmp_path / "box.obj", *R.box(o - s / 2, o + s * np.array([9, 13, 9]) + s / 2))
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    _run(_mini("dfsph") + ["--frames", "3", "--dump", a])
    _run(_mini("dfsph") + ["--frames", "3", "--dump", b, "--fluid-mesh", obj])
    for f in ("pos", "density"):
        assert np.array_equal(np.fromfile(a + f".{f}.f32", np.uint32), np.fromfile(b + f".{f}.f32", np.uint32)), f


@pytest.mark.parametrize("solver", SOLVERS)
def test_mesh_body_layers_agree(pkg, built, solver, tmp_path):
    """--mesh-body: sph_headless, capi.SphApp and engine.SphkSystem over four frames, bit for bit"""
    _gpu()
    import dataclasses
    from cpp_fluid_particles_b200 import capi, engine
    meshes = _m()
    obj = R.write_obj(tmp_path / "ico.obj", *R.icosphere(2, 0.05))
    spec = [obj + ",0.7,1,0.235,0.20,0.235"]
    prefix, dump = str(tmp_path / "scene"), str(tmp_path / "dump")
    _run(_mini(solver) + ["--mesh-body"] + spec + ["--emit-scene", prefix])
    res = _run(_mini(solver) + ["--mesh-body"] + spec + ["--frames", "4", "--dump", dump])
    body = meshes.load_obj(obj, 1.0, (0.235, 0.20, 0.235)).body(SB, 0.7)
    assert np.array_equal(bits(np.fromfile(prefix + ".body.f32", np.float32).reshape(-1, 3)), bits(body["points"]))
    dyn = np.fromfile(prefix + ".body_dyn.f32", np.float32)
    assert np.array_equal(bits(dyn), bits(np.float32([body["mass"], *body["inertia"]])))
    sc = pkg.scene.benchmark_scene("mini", solver)
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(np.fromfile(prefix + ".fluid.f32", np.float32).reshape(-1, 3)))
    app = capi.SphApp(sc, bodies=[body])
    e = engine.SphkSystem(sc, bodies=[body])
    try:
        for _ in range(4):
            app.step(); e.step()
        a = app.download()
        pos = np.fromfile(dump + ".pos.f32", np.float32).reshape(-1, 3)
        assert np.array_equal(bits(pos), bits(a["pos"])) and np.array_equal(bits(pos), bits(e.state()["pos"]))
        for got in (app.body_pose(0), e.body_pose()[0]):
            assert np.array_equal(bits(got), bits(np.float32(res["body_pose"])))
        assert np.array_equal(bits(app.body_motion(0)), bits(np.float32(res["body_motion"])))
        assert np.array_equal(bits(app.body_impulse(0)), bits(np.float32(res["body_impulse"])))
        assert np.array_equal(bits(e.body_impulse()[0]), bits(np.float32(res["body_impulse"])))
    finally:
        app.close(); e.close()


def test_rotated_body_samples_on_its_mesh(pkg, built):
    """an asymmetric box, rotated: after placement (step 0) its particles lie on the world-space mesh"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    meshes = _m()
    q = np.array([0.2, 0.4, -0.3, 0.8]); q /= np.linalg.norm(q)
    x, y, z, w = q
    Rq = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    v, f = R.box((-0.06, -0.03, -0.045), (0.06, 0.03, 0.045))
    m = meshes.Mesh((v @ Rq.T + [0.25, 0.3, 0.25]).astype(np.float32), f)
    body = m.body(SB, 0.0)
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    app = capi.SphApp(sc, bodies=[body])
    try:
        b = app.download_boundary()["pos"]                 # (in the search's order: the body's particles among the shell's)
        assert len(b) == len(sc.boundary) + len(body["points"])
        assert np.count_nonzero(m.classify(b, 1e-5) & 2) == len(body["points"])
    finally:
        app.close()


# ---- physics ------------------------------------------------------------------------------------------------------------------------
DAM = ["--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055", "0.135", "--quiet"]


@pytest.mark.parametrize("solver", SOLVERS)
def test_static_torus_obstacle_is_leak_tight(pkg, built, solver, tmp_path):
    _gpu()
    meshes = _m()
    obj = R.write_obj(tmp_path / "torus.obj", *R.torus(0.09, 0.035, 48, 24))
    t = (0.25, 0.09, 0.25)
    dump = str(tmp_path / "d")
    _run([CLI, "--solver", {"wcsph": "sph"}.get(solver, solver), "--frames", "400" if solver == "wcsph" else "100"] + DAM +
         ["--obstacle", f"{obj},1,{t[0]},{t[1]},{t[2]}", "--dump", dump])
    pos = np.fromfile(dump + ".pos.f32", np.float32).reshape(-1, 3)
    assert np.all(np.isfinite(pos))
    fl = meshes.load_obj(obj, 1.0, t).classify(pos, SB / 2)
    assert np.count_nonzero(fl) == 0, f"{np.count_nonzero(fl & 1)} inside, {np.count_nonzero(fl & 2)} within r/2"


def test_turning_torus_body_is_leak_tight(pkg, built, tmp_path):
    """a kinematic torus turning about x in the settling block (DFSPH): no fluid inside it or within r/2 after 100 frames"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    meshes = _m()
    m = meshes.Mesh(np.asarray(R.torus(0.08, 0.03, 48, 24)[0], np.float32), R.torus(0.08, 0.03, 48, 24)[1], 1.0, (0.25, 0.16, 0.25))
    body = m.body(SB, 0.0)
    body["angular_velocity"] = np.float32([2.0, 0.0, 0.0])
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    keep = m.classify(sc.fluid, SB) == 0
    import dataclasses
    sc = dataclasses.replace(sc, fluid=np.ascontiguousarray(sc.fluid[keep]))
    app = capi.SphApp(sc, bodies=[body])
    try:
        for _ in range(100):
            app.step()
        pose = app.body_pose(0).astype(np.float64)
        pos = app.download()["pos"]
    finally:
        app.close()
    x, y, z, w = pose[3:]
    Rq = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    # the mesh in its current pose: body frame from the properties, then the pose
    p = m.properties()
    x0, y0, z0, w0 = p["orientation"]
    R0 = np.array([[1 - 2 * (y0 * y0 + z0 * z0), 2 * (x0 * y0 - z0 * w0), 2 * (x0 * z0 + y0 * w0)],
                   [2 * (x0 * y0 + z0 * w0), 1 - 2 * (x0 * x0 + z0 * z0), 2 * (y0 * z0 - x0 * w0)],
                   [2 * (x0 * z0 - y0 * w0), 2 * (y0 * z0 + x0 * w0), 1 - 2 * (x0 * x0 + y0 * y0)]])
    local = (m.vertices.astype(np.float64) - p["centroid"]) @ R0
    now = meshes.Mesh((local @ Rq.T + pose[:3]).astype(np.float32), m.triangles)
    fl = now.classify(pos, SB / 2)
    assert np.count_nonzero(fl) == 0, f"{np.count_nonzero(fl & 1)} inside, {np.count_nonzero(fl & 2)} within r/2"
    assert abs(float(np.arccos(np.clip(abs(w), 0, 1))) * 2) > 0.1, "the torus must have turned"


def test_buoyancy_ordering(pkg, built, tmp_path):
    """icosphere bodies of REL 0.5, 1 and 2 in a resting pool end in that height order; the 0.5 body breaks the surface"""
    _gpu()
    obj = R.write_obj(tmp_path / "ico.obj", *R.icosphere(2, 0.04))
    y = {}
    for rel in (0.5, 1.0, 2.0):
        res = _run([CLI, "--solver", "dfsph", "--frames", "150", "--box", "0.5", "--block", "22", "9", "22", "--origin", "0.035", "0.035",
                    "0.035", "--quiet", "--mesh-body", f"{obj},{rel},1,0.25,0.12,0.25"])
        y[rel] = res["body_pose"][1]
    surface = 0.035 + 0.02 * 8
    assert y[0.5] > y[1.0] > y[2.0], y
    assert y[0.5] + 0.04 > surface, y


def test_obstacle_combinations_run_finite(pkg, built, tmp_path):
    _gpu()
    obj = R.write_obj(tmp_path / "torus.obj", *R.torus(0.08, 0.03, 32, 16))
    ob = ["--obstacle", f"{obj},1,0.25,0.09,0.25"]
    for extra in (["--adhesion", "150"], ["--heat", "1e-4,0", "--wall-temp", "1"], ["--cfl", "0.4"]):
        dump = str(tmp_path / "c")
        _run([CLI, "--solver", "dfsph", "--frames", "20"] + DAM + ob + extra + ["--dump", dump])
        assert np.all(np.isfinite(np.fromfile(dump + ".pos.f32", np.float32)))


def test_memcheck_mesh_options(pkg, built, tmp_path):
    """compute-sanitizer memcheck of the headless app with every mesh option (SPHK_SANITIZER=1, as the other memcheck runs)"""
    _gpu()
    if os.environ.get("SPHK_SANITIZER") != "1":
        pytest.skip("SPHK_SANITIZER=1 runs the sanitizer")
    import shutil
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    torus = R.write_obj(tmp_path / "torus.obj", *R.torus(0.06, 0.02, 24, 12))
    ico = R.write_obj(tmp_path / "ico.obj", *R.icosphere(1, 0.03))
    box = R.write_obj(tmp_path / "box.obj", *R.box((0.05, 0.05, 0.05), (0.45, 0.3, 0.45)))
    cmd = [exe, "--tool", "memcheck", "--error-exitcode", "9", CLI, "--solver", "dfsph", "--frames", "2", "--box", "0.5", "--quiet",
           "--obstacle", f"{torus},1,0.25,0.1,0.25", "--mesh-body", f"{ico},0.5,1,0.25,0.25,0.15", "--fluid-mesh", box]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                       env=dict(os.environ, SPHK_STEP_GRAPH="0"))
    assert r.returncode == 0 and "ERROR SUMMARY: 0 errors" in r.stdout, r.stdout[-4000:]
