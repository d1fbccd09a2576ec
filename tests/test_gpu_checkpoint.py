"""Checkpoints on the GPU (DESIGN.md section 2.14): N steps, checkpoint, a fresh system restores, M more steps give the same bits as
N + M steps without stopping -- for every solver and every feature that keeps state -- plus the graph, non-interference, snapshot
time, refusal and device checksum cases."""
import dataclasses
import os

import numpy as np
import pytest

import checkpoint_ref as CR
import open_boundary_ref as OB
from util import bits

pytestmark = pytest.mark.gpu

F = np.float32
SPACING = 0.02
N_STEPS, M_STEPS = 7, 6


def _n(solver, case):
    """steps before the checkpoint in the resume matrix: about 0.2 s of simulated time, so that the block has reached the floor --
    warm stiffnesses are non-zero and the heated wall has touched the fluid (the step counts of frames for an adaptive run)"""
    if case == "adaptive":
        return 20
    return 200 if solver == "wcsph" else 50


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")


def _cube(side_pts, h=SPACING):
    a = (np.arange(side_pts) - 0.5 * (side_pts - 1)) * h
    p = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    return p[(np.abs(p) > a.max() - 1e-9).any(1)].astype(F)


def _body(position, w=(0, 0, 0), mass=None):
    b = {"points": _cube(4), "position": [float(x) for x in position], "orientation": [0.0, 0.0, 0.0, 1.0],
         "linear_velocity": [0.0, 0.0, 0.0], "angular_velocity": [float(x) for x in w]}
    if mass is not None:
        b["mass"], b["inertia"] = float(mass), [float(mass * 0.08 * 0.08 / 6)] * 3
    return b


def _scene(pkg, solver):
    if solver == "dfsph":       # adaptive thresholds, device loops (the facade's default)
        return pkg.scene.make_scene("mini", "dfsph", dt=0.004)
    return pkg.scene.benchmark_scene("mini", solver)


SCENES = ["plain", "vorticity", "stir", "float", "implicit_viscosity", "rheology", "heat", "adhesion", "tap_drain", "adaptive",
          "probes"]
PROBES = dict(points=[(0.2, 0.1, 0.2), (0.25, 0.2, 0.25)], gauges=[((0.235, 0.45, 0.235), (0.235, 0.0, 0.235))])


def _make(pkg, solver, case):
    """a configured facade system of the case (the same every call: the configuration a restore needs)"""
    from cpp_fluid_particles_b200 import capi
    sc = _scene(pkg, solver)
    if case == "stir":
        app = capi.SphApp(sc, bodies=[_body((0.235, 0.40, 0.235), w=(0.0, 3.0, 0.0))])
    elif case == "float":
        app = capi.SphApp(sc, bodies=[_body((0.235, 0.40, 0.235), mass=0.3)])
    elif case == "tap_drain":
        box, block, origin = pkg.scene._CONFIGS["mini"]
        e, sink = OB.tap_and_drain((box,) * 3, block, origin, 1.5, 0.2)
        app = capi.SphApp(sc, max_fluid=2 * sc.fluid.shape[0], emitters=[e], sinks=[(sink[:3], sink[3:])])
    else:
        app = capi.SphApp(sc)
    if case == "vorticity":
        app.set_vorticity(0.3)
    elif case == "implicit_viscosity":
        app.set_implicit_viscosity(0.05, 0.03)
    elif case == "rheology":
        app.set_rheology(dict(model="hb", k=0.02, n=0.6, tau_y=0.05, nu_max=0.5))
    elif case == "heat":
        app.set_thermal(dict(alpha=1e-3, beta=0.01, t_ref=20.0, wall=(80.0, 1.0)))
        app.set_thermal_viscosity(dict(nu_ref=0.01, e=0.02, nu_max=0.1))
    elif case == "adhesion":
        app.set_adhesion(dict(wall=150.0))
    elif case == "adaptive":
        app.set_adaptive_dt(0.4)
    elif case == "probes":
        app.set_probes(**PROBES)
    return app


def _advance(app, case, k):
    for _ in range(k):
        if case == "adaptive":
            app.advance(0.01)
        else:
            app.step()


def _state(app, case):
    s = dict(app.download())
    s.update({"b_" + k: v for k, v in app.download_boundary().items()})
    if case == "heat":
        s["temperature"] = app.download_temperature()
    if case in ("stir", "float"):
        s["pose"], s["motion"], s["impulse"] = app.body_pose(0), app.body_motion(0), app.body_impulse(0)
    if case == "tap_drain":
        st, chk = app.open_boundary_stats()
        s["open"] = np.array([st["emitted"], st["removed"], st["refused"], chk], np.int64)
    if case == "adaptive":
        a = app.adaptive_stats()
        s["adaptive"] = np.array([a["speed"], a["last_dt"], a["simulated_time"]], np.float64)
        s["counts"] = np.array([a["min_clamps"], a["nonfinite_steps"], a["source"]], np.int64)
    return s


def _same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.shape == y.shape and np.array_equal(bits(x), bits(y)), f"{what}: {k} differs"


def _series_tail(app, m):
    s = app.probe_series()
    return {k: s[k][-m:] for k in ("steps", "times", "records", "levels")}


# ---- the resume matrix -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", SCENES)
@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
def test_resume_matrix(pkg, built, tmp_path, solver, case):
    _gpu()
    path = str(tmp_path / "run.ckpt")
    n = _n(solver, case)
    a = _make(pkg, solver, case)
    _advance(a, case, n + M_STEPS)
    want = _state(a, case)
    want_rows = _series_tail(a, M_STEPS) if case == "probes" else None
    a.close()
    b = _make(pkg, solver, case)
    _advance(b, case, n)
    b.checkpoint(path, b"frame 7")
    b.checkpoint_wait()
    b.close()
    c = _make(pkg, solver, case)
    assert c.restore(path) == b"frame 7"
    _advance(c, case, M_STEPS)
    _same(want, _state(c, case), f"{solver}/{case}")
    if case == "probes":
        got = _series_tail(c, M_STEPS)
        _same(want_rows, got, f"{solver}/{case} probe rows")
        assert list(got["steps"]) == list(range(n + 1, n + M_STEPS + 1))
    c.close()


def test_resume_at_the_bench_scene(pkg, built, tmp_path):
    """the 2M-particle DFSPH benchmark scene, a few steps on either side"""
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("2m", "dfsph")
    path = str(tmp_path / "big.ckpt")
    a = capi.SphApp(sc)
    for _ in range(3):
        a.step()
    a.checkpoint(path)
    for _ in range(3):
        a.step()
    want = _state(a, "plain")
    a.checkpoint_wait()
    a.close()
    c = capi.SphApp(sc)
    c.restore(path)
    for _ in range(3):
        c.step()
    _same(want, _state(c, "plain"), "2M DFSPH")
    c.close()


# ---- graph, non-interference, snapshot time ------------------------------------------------------------------------------------
@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
def test_checkpoint_every_step_changes_nothing_and_keeps_the_graph(pkg, built, tmp_path, solver):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", solver)
    plain, ck = capi.SphApp(sc), capi.SphApp(sc)
    for k in range(10):
        plain.step(); ck.step()
        was = ck.step_graph_active()
        ck.checkpoint(str(tmp_path / "every.ckpt"))
        assert ck.step_graph_active() == was
    ck.checkpoint_wait()
    assert ck.step_graph_active()
    _same(_state(plain, "plain"), _state(ck, "plain"), solver)
    plain.close(); ck.close()


@pytest.mark.parametrize("direction", ["graph_to_plain", "plain_to_graph"])
def test_graph_and_plain_runs_resume_each_other(pkg, built, tmp_path, direction):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    path = str(tmp_path / "g.ckpt")
    src_graph = direction == "graph_to_plain"
    a = capi.SphApp(sc)
    a.set_option(3, 1 if src_graph else 0)
    for _ in range(N_STEPS):
        a.step()
    assert a.step_graph_active() == src_graph
    a.checkpoint(path)
    a.checkpoint_wait()
    for _ in range(M_STEPS):
        a.step()
    want = _state(a, "plain")
    a.close()
    c = capi.SphApp(sc)
    c.set_option(3, 0 if src_graph else 1)
    c.restore(path)
    for _ in range(M_STEPS):
        c.step()
    _same(want, _state(c, "plain"), direction)
    c.close()


def test_the_snapshot_is_the_state_at_the_call(pkg, built, tmp_path):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "dfsph")
    path = str(tmp_path / "t.ckpt")
    a = capi.SphApp(sc)
    for _ in range(N_STEPS):
        a.step()
    at_n = _state(a, "plain")
    a.checkpoint(path)
    for _ in range(M_STEPS):       # enqueued before the wait: they overwrite the arrays while the copy may still run
        a.step()
    a.checkpoint_wait()
    a.close()
    c = capi.SphApp(sc)
    c.restore(path)
    _same(at_n, _state(c, "plain"), "snapshot")
    c.close()


# ---- the file against the numpy reader -----------------------------------------------------------------------------------------
def test_file_parses_with_the_reference_and_holds_the_api_arrays(pkg, built, tmp_path):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.benchmark_scene("mini", "pbd")
    path = tmp_path / "p.ckpt"
    a = capi.SphApp(sc)
    for _ in range(3):
        a.step()
    a.checkpoint(str(path), b"abc")
    a.checkpoint_wait()
    st = a.download()
    f = CR.parse(path.read_bytes())
    sec = f["sections"]
    assert f["config"]["solver"] == "pbd" and f["config"]["capacity_fluid"] == st["pos"].shape[0]
    assert sec["fluid.pos"]["data"] == st["pos"].tobytes() and sec["fluid.vel"]["data"] == st["vel"].tobytes()
    assert sec["fluid.particle2cell"]["data"] == st["p2c"].tobytes() and sec["user"]["data"] == b"abc"
    assert "solver.pbd_pos_last" in sec and "system.record" in sec
    assert not os.path.exists(str(path) + ".tmp")
    a.close()


# ---- refusals: the state compared array by array before and after --------------------------------------------------------------
def _printed(capfd) -> str:
    import ctypes as C
    C.CDLL(None).fflush(None)        # the library prints through C stdio
    return capfd.readouterr().out


def _refused(app, path, case="plain", capfd=None, names=None):
    """restore refused, the state unchanged array by array, and (with capfd) the printed reason naming `names`"""
    before = _state(app, case)
    if capfd is not None:
        _printed(capfd)
    with pytest.raises(RuntimeError):
        app.restore(str(path))
    if capfd is not None:
        out = _printed(capfd)
        assert names in out, out
    _same(before, _state(app, case), "after a refused restore")


@pytest.fixture
def saved(pkg, built, tmp_path):
    _gpu()
    from cpp_fluid_particles_b200 import capi
    sc = pkg.scene.make_scene("mini", "dfsph", dt=0.004)
    path = tmp_path / "s.ckpt"
    a = capi.SphApp(sc)
    a.set_adhesion(dict(wall=150.0))
    for _ in range(4):
        a.step()
    a.checkpoint(str(path))
    a.checkpoint_wait()
    a.close()
    return sc, path


@pytest.mark.parametrize("what, names", [("dt", "config: dt differs"), ("solver", "config: solver differs"),
                                         ("capacity", "config: capacity_fluid differs"), ("adhesion_beta", "config: settings differ"),
                                         ("bodies", "config: capacity_boundary differs")])
def test_a_fingerprint_mismatch_is_refused(pkg, saved, capfd, what, names):
    from cpp_fluid_particles_b200 import capi
    sc, path = saved
    if what == "dt":
        sc = dataclasses.replace(sc, params=dataclasses.replace(sc.params, dt=0.003))
    elif what == "solver":
        sc = pkg.scene.make_scene("mini", "wcsph", dt=0.004)
    kw = {}
    if what == "capacity":
        kw = dict(max_fluid=sc.fluid.shape[0] + 10, emitters=[], sinks=[])
    elif what == "bodies":
        kw = dict(bodies=[_body((0.235, 0.40, 0.235))])
    app = capi.SphApp(sc, **kw)
    app.set_adhesion(dict(wall=149.0 if what == "adhesion_beta" else 150.0))
    app.step()
    _refused(app, path, capfd=capfd, names=names)
    app.close()


@pytest.mark.parametrize("case", ["adhesion", "float", "tap_drain"])
def test_a_flipped_payload_bit_in_any_section_is_refused(pkg, built, tmp_path, capfd, case):
    """every section, the library's body and open-boundary sections included; the printed reason names the section"""
    _gpu()
    path = tmp_path / "s.ckpt"
    a = _make(pkg, "dfsph", case)
    _advance(a, case, 20)
    a.checkpoint(str(path))
    a.checkpoint_wait()
    a.close()
    data = path.read_bytes()
    f = CR.parse(data)
    names = set(f["sections"])
    if case == "float":
        assert {"ctx.body_pose", "ctx.body_motion", "ctx.body_impulse", "ctx.body_local", "ctx.body_decl"} <= names
    if case == "tap_drain":
        assert {"ctx.open_check", "system.emitter_carry"} <= names
    app = _make(pkg, "dfsph", case)
    app.step()
    for name, sec in f["sections"].items():
        if sec["bytes"] == 0:
            continue
        b = bytearray(data)
        b[sec["offset"] + sec["bytes"] // 2] ^= 0x10
        bad = tmp_path / "flip.ckpt"
        bad.write_bytes(bytes(b))
        _refused(app, bad, case, capfd, f"section '{name}': checksum mismatch")
    app.restore(str(path))        # the good file still restores
    app.close()


@pytest.mark.parametrize("what", ["truncated", "version"])
def test_truncated_and_wrong_version_are_refused(saved, tmp_path, what):
    from cpp_fluid_particles_b200 import capi
    sc, path = saved
    data = path.read_bytes()
    bad = tmp_path / "bad.ckpt"
    bad.write_bytes(data[:-7] if what == "truncated" else CR.with_header(data, version=9))
    app = capi.SphApp(sc)
    app.set_adhesion(dict(wall=150.0))
    app.step()
    _refused(app, bad)
    app.close()


def test_an_unwritable_path_keeps_the_previous_file(saved, tmp_path):
    from cpp_fluid_particles_b200 import capi
    sc, path = saved
    good = path.read_bytes()
    app = capi.SphApp(sc)
    app.set_adhesion(dict(wall=150.0))
    app.step()
    missing = tmp_path / "no_such_dir" / "x.ckpt"
    app.checkpoint(str(missing))
    with pytest.raises(RuntimeError):
        app.checkpoint_wait()
    if os.geteuid() == 0:         # a read-only directory does not stop root: the first half stands alone
        app.close()
        return
    os.chmod(tmp_path, 0o500)
    try:
        app.checkpoint(str(path))
        with pytest.raises(RuntimeError):
            app.checkpoint_wait()
    finally:
        os.chmod(tmp_path, 0o700)
    assert path.read_bytes() == good
    app.close()


def test_on_demand_probes_wait_for_a_step_after_restore(saved):
    from cpp_fluid_particles_b200 import capi
    sc, path = saved
    app = capi.SphApp(sc)
    app.set_adhesion(dict(wall=150.0))
    for _ in range(30):           # last-step statistics that are not zero before the restore
        app.step()
    assert app.dfsph_iterations() != (0, 0) and app.adhesion_stats()["wetted"] > 0
    app.restore(str(path))
    with pytest.raises(RuntimeError):
        app.sample_probes([(0.2, 0.1, 0.2)])
    with pytest.raises(RuntimeError):
        app.sample_lattice((0.1, 0.1, 0.1), 0.05, (2, 2, 2))
    assert app.dfsph_iterations() == (0, 0) and app.adhesion_stats()["wetted"] == 0
    app.step()
    assert app.sample_probes([(0.2, 0.1, 0.2)]).shape == (1, 8)
    app.close()


# ---- the device checksum -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 4095, 4096, 8 * (1 << 24) + 24])
@pytest.mark.parametrize("offset", [0, 4])
def test_device_checksum_equals_the_reference(pkg, built, n, offset):
    """16-byte and unaligned sources; the last size is a section of more than 2^24 words, beyond one block's reach"""
    _gpu()
    import ctypes as C
    import torch
    from cpp_fluid_particles_b200 import capi, engine
    if n > 1 << 20 and offset:
        pytest.skip("one large case suffices")
    g = torch.Generator(device="cuda").manual_seed(n)
    buf = torch.randint(0, 256, (n + 16,), dtype=torch.uint8, device="cuda", generator=g)
    s = engine.SphkSystem(pkg.scene.make_scene("mini"), step0=False)
    L = capi.sphk()
    out = C.c_ulonglong(0)
    L.sphk_state_checksum_device.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.POINTER(C.c_ulonglong)]
    assert L.sphk_state_checksum_device(s.ctx, C.c_void_p(buf.data_ptr() + offset), n, C.byref(out)) == 0
    host = buf.cpu().numpy().tobytes()[offset:offset + n]
    assert out.value == CR.checksum(host)
    s.close()



# ---- layer crossings: a file of one layer restores in the other ---------------------------------------------------------------
def _engine(pkg, solver, case):
    """the python engine configured as _make configures the facade"""
    from cpp_fluid_particles_b200 import engine
    sc = _scene(pkg, solver)
    kw = {}
    if case == "float":
        kw = dict(bodies=[_body((0.235, 0.40, 0.235), mass=0.3)])
    elif case == "tap_drain":
        box, block, origin = pkg.scene._CONFIGS["mini"]
        e, sink = OB.tap_and_drain((box,) * 3, block, origin, 1.5, 0.2)
        kw = dict(max_fluid=2 * sc.fluid.shape[0], emitters=[e], sinks=[(sink[:3], sink[3:])])
    s = engine.SphkSystem(sc, **kw)
    if case == "adhesion":
        s.adhesion = dict(wall=150.0)
    elif case == "heat":
        s.thermal = dict(alpha=1e-3, beta=0.01, t_ref=20.0, wall=(80.0, 1.0))
        s.thermal_viscosity = dict(nu_ref=0.01, e=0.02, nu_max=0.1)
    elif case == "vorticity":
        s.vorticity_eps = 0.3
    return s


def _core(st):
    """the arrays both layers return"""
    return {k: np.asarray(st[k]) for k in ("pos", "vel", "density", "pressure", "mass", "p2c")}


CROSSINGS = [("wcsph", "plain"), ("dfsph", "plain"), ("pbd", "plain"), ("dfsph", "adhesion"), ("pbd", "vorticity"),
             ("dfsph", "float"), ("pbd", "tap_drain"), ("wcsph", "heat")]


@pytest.mark.parametrize("solver, case", CROSSINGS)
@pytest.mark.parametrize("direction", ["class_to_engine", "engine_to_class"])
def test_files_cross_layers(pkg, built, tmp_path, direction, solver, case):
    _gpu()
    n, path = 30, str(tmp_path / "x.ckpt")
    a = _make(pkg, solver, case)
    _advance(a, case, n + M_STEPS)
    want = _core(a.download())
    a.close()
    if direction == "class_to_engine":
        b = _make(pkg, solver, case)
        _advance(b, case, n)
        b.checkpoint(path, b"cross")
        b.checkpoint_wait()
        b.close()
        c = _engine(pkg, solver, case)
        assert c.load_state(path) == b"cross"
        for _ in range(M_STEPS):
            c.step()
        got = _core(c.state())
        c.close()
    else:
        b = _engine(pkg, solver, case)
        for _ in range(n):
            b.step()
        b.save_state(path, b"cross")
        b.wait_state()
        b.close()
        c = _make(pkg, solver, case)
        assert c.restore(path) == b"cross"
        _advance(c, case, M_STEPS)
        got = _core(c.download())
        c.close()
    _same(want, got, f"{direction} {solver}/{case}")


# ---- the headless app: 20 frames against 10 + checkpoint, then a resume to 20 -------------------------------------------------------
def test_headless_round_trip(built, tmp_path):
    _gpu()
    import json
    import subprocess
    from util import ROOT
    cli = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
    scene = ["--solver", "dfsph", "--box", "0.5", "--block", "10", "14", "10", "--origin", "0.135", "0.055", "0.135", "--quiet",
             "--probe", "0.2,0.1,0.2", "--gauge", "0.235,0.002,0.235,0.235,0.45,0.235"]
    t = str(tmp_path)

    def run(*extra):
        r = subprocess.run([cli] + scene + list(extra), stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)
        assert r.returncode == 0, r.stderr + r.stdout
        return json.loads(r.stdout.strip().splitlines()[-1])

    run("--frames", "20", "--dump", t + "/a", "--probe-out", t + "/a.csv")
    first = run("--frames", "10", "--checkpoint", t + "/run.ckpt", "--checkpoint-every", "4", "--probe-out", t + "/b.csv")
    assert first["checkpoints_written"] == 3 and first["resumed_from_frame"] == -1
    second = run("--frames", "20", "--resume", t + "/run.ckpt", "--dump", t + "/b", "--probe-out", t + "/b.csv")
    assert second["resumed_from_frame"] == 10 and second["frames"] == 20
    for suffix in (".pos.f32", ".rgb.f32", ".density.f32"):
        assert open(t + "/a" + suffix, "rb").read() == open(t + "/b" + suffix, "rb").read(), suffix
    assert open(t + "/a.csv", "rb").read() == open(t + "/b.csv", "rb").read()
