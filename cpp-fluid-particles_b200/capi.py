"""ctypes bindings of the two in-tree native libraries.

  libsphk.so     the C-ABI of include/sphk.h (CUDA kernels, sm_90a)
  libsphhost.so  the reference-shaped C++ classes + headless facade of include/sph_app.h

There is no CPU fallback anywhere in this package: a missing library raises ImportError-like
RuntimeError immediately, and sphk_create fails with SPHK_ERR_NO_DEVICE on a box without a GPU.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIBSPHK = os.path.join(HERE, "libsphk.so")
LIBHOST = os.path.join(HERE, "libsphhost.so")

SPHK_FUNCTIONS = [
    "sphk_create", "sphk_destroy", "sphk_set_option", "sphk_set_grid", "sphk_synchronize", "sphk_error_string", "sphk_launch_count",
    "sphk_device_rcp", "sphk_neighbor_search", "sphk_permute", "sphk_refresh", "sphk_boundary_mass", "sphk_fill",
    "sphk_gravity", "sphk_viscosity", "sphk_color_grad", "sphk_surface", "sphk_density", "sphk_pressure",
    "sphk_pressure_force", "sphk_advect", "sphk_dfsph_density_alpha", "sphk_dfsph_div_error", "sphk_dfsph_div_correct",
    "sphk_dfsph_den_error", "sphk_dfsph_den_correct", "sphk_reduce_abs_sum", "sphk_copy", "sphk_pbd_density_lambda",
    "sphk_pbd_delta_pos_apply", "sphk_pbd_velocity_from_positions", "sphk_pbd_xsph", "sphk_get_permutation",
    "sphk_list_stats", "sphk_get_skin_displacement", "sphk_set_active_range", "sphk_push_range", "sphk_build_neighbor_list", "sphk_get_neighbor_list", "sphk_get_tile_lists", "sphk_fused_density_color_grad",
    "sphk_fused_dfsph_density_alpha_color_grad", "sphk_fused_dfsph_density_alpha_div_error", "sphk_fused_pbd_xsph_color_grad", "sphk_scene_fluid_block", "sphk_scene_boundary_count", "sphk_scene_boundary_shell", "sphk_loop_begin", "sphk_loop_next", "sphk_loop_end", "sphk_loop_iterations", "sphk_fused_viscosity_surface", "sphk_vorticity", "sphk_vorticity_confinement",
    "sphk_fused_viscosity_surface_vorticity", "sphk_fused_pbd_xsph_vorticity", "sphk_export_dots", "sphk_particles_advect", "sphk_add_launches",
    "sphk_mg_unique_id", "sphk_mg_init", "sphk_mg_destroy", "sphk_mg_ipc_handle", "sphk_mg_ipc_connect", "sphk_mg_set_transport",
    "sphk_mg_exchange_ints", "sphk_mg_exchange_ints_async", "sphk_mg_plane_ranges", "sphk_mg_halo_device", "sphk_mg_check_async", "sphk_set_active_range_device", "sphk_mg_allreduce_sum", "sphk_mg_exchange_slices", "sphk_mg_halo", "sphk_mg_check", "sphk_mg_stats",
    "sphk_strays_block_floats", "sphk_strays_collect", "sphk_strays_append", "sphk_mg_strays_route", "sphk_strays_counts",
    "sphk_bodies_init", "sphk_bodies_set_motion", "sphk_bodies_step", "sphk_bodies_get_pose", "sphk_bodies_get_local",
    "sphk_bodies_set_dynamics", "sphk_bodies_react", "sphk_bodies_integrate", "sphk_bodies_set_body_motion",
    "sphk_bodies_get_motion", "sphk_bodies_get_impulse",
    "sphk_implicit_viscosity_work_floats", "sphk_implicit_viscosity", "sphk_implicit_viscosity_stats", "sphk_visc_implicit_setup",
    "sphk_visc_implicit_matvec",
    "sphk_emitter_axes", "sphk_emitter_advance", "sphk_emit", "sphk_sinks_apply", "sphk_sinks_removed", "sphk_fluid_set_count",
    "sphk_open_check", "sphk_time_step", "sphk_step_speed", "sphk_step_speed_result",
]
SPH_APP_FUNCTIONS = [
    "sph_app_create", "sph_app_destroy", "sph_app_step", "sph_app_fluid_size", "sph_app_boundary_size",
    "sph_app_download_fluid", "sph_app_download_boundary", "sph_app_upload_fluid", "sph_app_engine",
    "sph_app_submit", "sph_app_wait", "sph_app_dfsph_iterations", "sph_app_set_option", "sph_app_set_vorticity",
    "sph_app_create_with_bodies", "sph_app_set_body_motion", "sph_app_body_pose", "sph_app_step_graph_active",
    "sph_app_create_with_dynamic_bodies", "sph_app_body_motion", "sph_app_body_impulse", "sph_app_set_implicit_viscosity",
    "sph_app_viscosity_stats", "sph_app_create_open", "sph_app_open_boundary_stats", "sph_app_set_adaptive_dt", "sph_app_advance",
    "sph_app_adaptive_stats",
]

OPT_NEIGHBOR_LIST, OPT_LIST_CAPACITY, OPT_LIST_SKIN, OPT_SIMPLE_LIST_BUILD, OPT_TILE, OPT_STAGED_LIST_BUILD, OPT_PATCH = 1, 2, 5, 6, 9, 10, 11
MAX_EMITTERS, MAX_SINKS = 16, 16   # SPHK_MAX_EMITTERS, SPHK_MAX_SINKS
DT_MIN_CLAMP, DT_NONFINITE, DT_FRAME_END = 1, 2, 4   # SPHK_DT_* flags of sphk_time_step
# tile-list geometry of csrc/sphk_internal.cuh (SPHK_BLOCK, SPHK_TILE_WINS, SPHK_TILE_CAP): sphk_get_tile_lists copies
# TILE_WINDOWS windows per tile of TILE_PARTICLES particles; a tile whose windows exceed TILE_CAP records walks the cells
TILE_PARTICLES, TILE_WINDOWS, TILE_CAP = 128, 18, 1535


def body_mass_inertia(bodies) -> np.ndarray:
    """{M, Ix, Iy, Iz} per body from the body dicts' optional "mass" (default 0: kinematic) and "inertia" (default 0)."""
    return np.ascontiguousarray([[float(b.get("mass", 0.0)), *[float(x) for x in b.get("inertia", (0.0, 0.0, 0.0))]]
                                 for b in bodies], np.float32).reshape(-1, 4)


class SphkEmitter(C.Structure):
    """sphk_emitter (include/sphk.h); sph_app_emitter has the same layout."""
    _fields_ = [("origin", C.c_float * 3), ("direction", C.c_float * 3), ("speed", C.c_float), ("spacing", C.c_float),
                ("width", C.c_int), ("height", C.c_int)]


def emitter_struct(e: dict) -> SphkEmitter:
    """An emitter dict {"origin", "direction", "speed", "spacing", "width", "height"} as the C struct."""
    k = SphkEmitter()
    k.origin[:] = [float(x) for x in e["origin"]]
    k.direction[:] = [float(x) for x in e["direction"]]
    k.speed, k.spacing = float(e["speed"]), float(e["spacing"])
    k.width, k.height = int(e.get("width", 1)), int(e.get("height", 1))
    return k


def sink_boxes(sinks) -> np.ndarray:
    """[(lo, hi), ...] as float32 {lo.xyz, hi.xyz} rows."""
    return np.ascontiguousarray([[*lo, *hi] for lo, hi in sinks], np.float32).reshape(-1, 6)


class SphkTimeStepRule(C.Structure):
    """sphk_time_step_rule (include/sphk.h)."""
    _fields_ = [("cfl", C.c_double), ("dt_min", C.c_double), ("dt_max", C.c_double), ("radius", C.c_double), ("gravity", C.c_double)]


class SphkGrid(C.Structure):
    _fields_ = [("cell_size", C.c_int * 3), ("cell_length", C.c_float), ("origin", C.c_int * 3)]


class SphkParticles(C.Structure):
    _fields_ = [("pos", C.c_void_p), ("vel", C.c_void_p), ("mass", C.c_void_p), ("density", C.c_void_p),
                ("pressure", C.c_void_p), ("particle2cell", C.c_void_p), ("n", C.c_int)]


class SphkScene(C.Structure):
    _fields_ = [("fluid", SphkParticles), ("boundary", SphkParticles), ("cell_start_fluid", C.c_void_p),
                ("cell_start_boundary", C.c_void_p), ("radius", C.c_float)]


class SphAppParams(C.Structure):
    _fields_ = [("space", C.c_float * 3), ("cell_length", C.c_float), ("radius", C.c_float), ("dt", C.c_float),
                ("m0", C.c_float), ("rho0", C.c_float), ("rho_boundary", C.c_float), ("stiff", C.c_float),
                ("visc", C.c_float), ("surface_tension", C.c_float), ("air_pressure", C.c_float),
                ("gravity", C.c_float * 3), ("cell_size", C.c_int * 3), ("solver", C.c_int), ("max_iter", C.c_int),
                ("density_error_threshold", C.c_float), ("divergence_error_threshold", C.c_float)]


_sphk = None
_apps = {}


def _load(path: str):
    if not os.path.exists(path):
        raise RuntimeError(f"{os.path.basename(path)} is not built ({path}); run __graft_entry__.build() -- "
                           "this package has no CPU or pure-python fallback")
    # RTLD_LOCAL: libsphhost.so and the reference build oracle/_ref/libsphref.so export the SAME C++ class
    # symbols (SPHSystem::step, ...) by design; they must never interpose each other in one process
    return C.CDLL(path, mode=C.RTLD_LOCAL)


def sphk():
    """libsphk.so with argument/return types set."""
    global _sphk
    if _sphk is None:
        L = _load(LIBSPHK)
        L.sphk_error_string.restype = C.c_char_p
        L.sphk_launch_count.restype = C.c_longlong
        L.sphk_scene_boundary_count.restype = C.c_longlong
        L.sphk_strays_block_floats.restype = C.c_longlong
        L.sphk_implicit_viscosity_work_floats.restype = C.c_longlong
        L.sphk_destroy.restype = None
        L.sphk_mg_destroy.restype = None
        _sphk = L
    return _sphk


def app_lib(path: str = LIBHOST):
    """A library exporting the sph_app_* facade: libsphhost.so (product) or oracle/_ref/libsphref.so."""
    if path not in _apps:
        if path == LIBHOST:
            sphk()
        L = _load(path)
        L.sph_app_create.restype = C.c_void_p
        L.sph_app_create_with_bodies.restype = C.c_void_p
        L.sph_app_create_with_dynamic_bodies.restype = C.c_void_p
        L.sph_app_create_open.restype = C.c_void_p
        L.sph_app_step.restype = C.c_float
        L.sph_app_engine.restype = C.c_char_p
        L.sph_app_destroy.restype = None
        _apps[path] = L
    return _apps[path]


def check(rc: int, what: str = "sphk"):
    if rc != 0:
        raise RuntimeError(f"{what} failed: {sphk().sphk_error_string(C.c_int(rc)).decode()} ({rc})")


def app_params(p) -> SphAppParams:
    """SceneParams (scene.py) -> sph_app_params."""
    q = SphAppParams()
    q.space[:] = [float(x) for x in p.space]
    q.cell_length, q.radius, q.dt, q.m0 = p.cell_length, p.radius, p.dt, p.m0
    q.rho0, q.rho_boundary, q.stiff, q.visc = p.rho0, p.rho_boundary, p.stiff, p.visc
    q.surface_tension, q.air_pressure = p.surface_tension, p.air_pressure
    q.gravity[:] = [float(x) for x in p.gravity]
    q.cell_size[:] = [int(x) for x in p.cell_size]
    q.solver, q.max_iter = p.solver_id, int(p.max_iter)
    q.density_error_threshold = p.density_error_threshold
    q.divergence_error_threshold = p.divergence_error_threshold
    return q


class SphApp:
    """One headless SPHSystem driven through the sph_app facade (numpy in / numpy out).

    `lib_path` selects the engine underneath: this repo's libsphhost.so (default) or the reference's own
    CUDA build oracle/_ref/libsphref.so -- the facade source is the same file for both."""

    def __init__(self, scene, lib_path: str = LIBHOST, bodies=None, max_fluid=None, emitters=None, sinks=None):
        """emitters / sinks / max_fluid: open boundaries (sph_app_create_open; engine.SphkSystem's format), no bodies.
        bodies: rigid bodies in engine.SphkSystem's format (sph_app_create_with_bodies; with a "mass" key on any body,
        sph_app_create_with_dynamic_bodies: dynamics are declared when some mass is > 0, as in engine.SphkSystem); their
        particles follow the static boundary set, so nB counts them."""
        self.L = app_lib(lib_path)
        self.scene = scene
        fl = np.ascontiguousarray(scene.fluid, np.float32)
        bd = np.ascontiguousarray(scene.boundary, np.float32)
        self.nF, self.nB = fl.shape[0], bd.shape[0]
        prm = app_params(scene.params)
        if emitters is not None or sinks is not None:
            em = list(emitters or [])
            ems = (SphkEmitter * max(1, len(em)))(*[emitter_struct(e) for e in em])
            boxes = sink_boxes(sinks or [])
            cap = int(max_fluid) if max_fluid is not None else self.nF
            self.h = self.L.sph_app_create_open(fl.ctypes.data_as(C.c_void_p), C.c_int(self.nF), C.c_int(cap),
                                                bd.ctypes.data_as(C.c_void_p), C.c_int(self.nB), C.c_int(len(em)), ems,
                                                C.c_int(boxes.shape[0]), boxes.ctypes.data_as(C.c_void_p), C.byref(prm))
        elif bodies is not None:     # (an empty list: the bodies constructor without bodies)
            pts = [np.asarray(b["points"], np.float32).reshape(-1, 3) for b in bodies]
            xyz = np.ascontiguousarray(np.concatenate(pts, 0) if pts else np.zeros((0, 3), np.float32))
            begin = np.ascontiguousarray(np.concatenate([[0], np.cumsum([len(q) for q in pts])]).astype(np.int32))
            pose = np.ascontiguousarray([[*b["position"], *b["orientation"]] for b in bodies], np.float32).reshape(-1, 7)
            motion = np.ascontiguousarray([[*b["linear_velocity"], *b["angular_velocity"]] for b in bodies], np.float32).reshape(-1, 6)
            self.nB += xyz.shape[0]
            args = [fl.ctypes.data_as(C.c_void_p), C.c_int(self.nF), bd.ctypes.data_as(C.c_void_p), C.c_int(bd.shape[0]),
                    C.c_int(len(bodies)), begin.ctypes.data_as(C.c_void_p), xyz.ctypes.data_as(C.c_void_p),
                    pose.ctypes.data_as(C.c_void_p), motion.ctypes.data_as(C.c_void_p)]
            if any("mass" in b for b in bodies):
                mi = body_mass_inertia(bodies)
                self.h = self.L.sph_app_create_with_dynamic_bodies(*args, mi.ctypes.data_as(C.c_void_p), C.byref(prm))
            else:
                self.h = self.L.sph_app_create_with_bodies(*args, C.byref(prm))
        else:
            self.h = self.L.sph_app_create(fl.ctypes.data_as(C.c_void_p), C.c_int(self.nF), bd.ctypes.data_as(C.c_void_p),
                                           C.c_int(self.nB), C.byref(prm))
        if not self.h:
            raise RuntimeError("sph_app_create failed (no CUDA device? there is no CPU fallback)")
        self.h = C.c_void_p(self.h)

    @property
    def engine(self) -> str:
        return self.L.sph_app_engine().decode()

    def step(self) -> float:
        ms = float(self.L.sph_app_step(self.h))
        self.nF = int(self.L.sph_app_fluid_size(self.h))    # open boundaries change the live count
        return ms

    @property
    def fluid_count(self) -> int:
        return int(self.L.sph_app_fluid_size(self.h))

    def open_boundary_stats(self):
        """({"emitted", "removed", "refused"} cumulative particle counts, sticky count-check bits); synchronises."""
        st, bits = (C.c_longlong * 3)(), C.c_int(0)
        if self.L.sph_app_open_boundary_stats(self.h, st, C.byref(bits)):
            raise RuntimeError("sph_app_open_boundary_stats failed (reference engine)")
        return {"emitted": int(st[0]), "removed": int(st[1]), "refused": int(st[2])}, int(bits.value)

    def download(self) -> dict:
        self.nF = self.fluid_count
        out = {"pos": np.empty((self.nF, 3), np.float32), "vel": np.empty((self.nF, 3), np.float32),
               "density": np.empty(self.nF, np.float32), "pressure": np.empty(self.nF, np.float32),
               "mass": np.empty(self.nF, np.float32), "p2c": np.empty(self.nF, np.int32)}
        rc = self.L.sph_app_download_fluid(self.h, *[out[k].ctypes.data_as(C.c_void_p) for k in
                                                     ("pos", "vel", "density", "pressure", "mass", "p2c")])
        if rc:
            raise RuntimeError("sph_app_download_fluid failed")
        return out

    def download_into(self, pos=None, vel=None, density=None):
        """D2H into caller-provided (pinned) buffers; None skips a field."""
        def p(a):
            return C.c_void_p(a.ctypes.data) if a is not None else None
        rc = self.L.sph_app_download_fluid(self.h, p(pos), p(vel), p(density), None, None, None)
        if rc:
            raise RuntimeError("sph_app_download_fluid failed")

    def download_boundary(self) -> dict:
        out = {"pos": np.empty((self.nB, 3), np.float32), "mass": np.empty(self.nB, np.float32),
               "p2c": np.empty(self.nB, np.int32)}
        rc = self.L.sph_app_download_boundary(self.h, *[out[k].ctypes.data_as(C.c_void_p) for k in ("pos", "mass", "p2c")])
        if rc:
            raise RuntimeError("sph_app_download_boundary failed")
        return out

    def upload(self, pos=None, vel=None):
        def p(a):
            return C.c_void_p(a.ctypes.data) if a is not None else None
        if self.L.sph_app_upload_fluid(self.h, p(pos), p(vel)):
            raise RuntimeError("sph_app_upload_fluid failed")

    def submit(self, pos_in, vel_in, pos_out=None, vel_out=None, density_out=None):
        """Pipelined host-buffer step (include/sph_app.h): numpy arrays over pinned host memory."""
        def p(a):
            return C.c_void_p(a.ctypes.data) if a is not None else None
        if self.L.sph_app_submit(self.h, p(pos_in), p(vel_in), p(pos_out), p(vel_out), p(density_out)):
            raise RuntimeError("sph_app_submit failed")

    def wait(self):
        if self.L.sph_app_wait(self.h):
            raise RuntimeError("sph_app_wait failed")

    def dfsph_iterations(self):
        """(divergence, density) iteration counts of the last DFSPH step."""
        a, b = C.c_int(0), C.c_int(0)
        if self.L.sph_app_dfsph_iterations(self.h, C.byref(a), C.byref(b)):
            raise RuntimeError("sph_app_dfsph_iterations: not a DFSPH system of this engine")
        return int(a.value), int(b.value)

    def set_option(self, option: int, value: int):
        """1: device-side loop tests (adaptive DFSPH), 2: fused sweeps, 3: step graph."""
        if self.L.sph_app_set_option(self.h, C.c_int(option), C.c_int(value)):
            raise RuntimeError("sph_app_set_option failed")

    def set_vorticity(self, eps: float):
        """Vorticity confinement of strength eps in every following step (0: off).  Not on the reference engine."""
        if self.L.sph_app_set_vorticity(self.h, C.c_float(eps)):
            raise RuntimeError("sph_app_set_vorticity failed (reference engine, or eps < 0)")

    def set_implicit_viscosity(self, nu: float, nu_boundary: float = 0.0, tol: float = 1e-4, max_iter: int = 20):
        """Implicit viscosity in every following step (nu = 0: off).  Not on the reference engine."""
        if self.L.sph_app_set_implicit_viscosity(self.h, C.c_float(nu), C.c_float(nu_boundary), C.c_float(tol), C.c_int(max_iter)):
            raise RuntimeError("sph_app_set_implicit_viscosity failed (reference engine or invalid values)")

    def viscosity_stats(self):
        """(iterations, relative residual) of the last implicit viscosity solve."""
        it, res = C.c_int(0), C.c_float(0.0)
        if self.L.sph_app_viscosity_stats(self.h, C.byref(it), C.byref(res)):
            raise RuntimeError("sph_app_viscosity_stats failed (reference engine)")
        return int(it.value), float(res.value)

    def set_body_motion(self, body: int, linear_velocity, angular_velocity):
        """New motion of one kinematic body from the next step on.  Not on the reference engine."""
        v = np.ascontiguousarray(linear_velocity, np.float32)
        w = np.ascontiguousarray(angular_velocity, np.float32)
        if self.L.sph_app_set_body_motion(self.h, C.c_int(body), v.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_set_body_motion failed (reference engine, bad index or non-finite motion)")

    def set_adaptive_dt(self, cfl: float, dt_min: float = 0.0, dt_max: float = 0.0):
        """CFL-adaptive time stepping from the next step on (cfl = 0: off).  Not on the reference engine."""
        if self.L.sph_app_set_adaptive_dt(self.h, C.c_float(cfl), C.c_float(dt_min), C.c_float(dt_max)):
            raise RuntimeError("sph_app_set_adaptive_dt failed (reference engine or invalid values)")

    def advance(self, frame_seconds: float):
        """CFL substeps until frame_seconds of simulated time have passed: (substeps, smallest dt)."""
        k, m = C.c_int(0), C.c_float(0.0)
        if self.L.sph_app_advance(self.h, C.c_double(frame_seconds), C.byref(k), C.byref(m)):
            raise RuntimeError("sph_app_advance failed (not adaptive, invalid frame or reference engine)")
        self.nF = self.fluid_count
        return int(k.value), float(m.value)

    def adaptive_stats(self) -> dict:
        """{"speed", "last_dt", "frame_min_dt", "source", "min_clamps", "nonfinite_steps", "simulated_time"}"""
        f, src, cnt, t = (C.c_float * 3)(), C.c_int(0), (C.c_longlong * 2)(), C.c_double(0.0)
        if self.L.sph_app_adaptive_stats(self.h, f, C.byref(src), cnt, C.byref(t)):
            raise RuntimeError("sph_app_adaptive_stats failed (reference engine)")
        return {"speed": float(f[0]), "last_dt": float(f[1]), "frame_min_dt": float(f[2]), "source": int(src.value),
                "min_clamps": int(cnt[0]), "nonfinite_steps": int(cnt[1]), "simulated_time": float(t.value)}

    def step_graph_active(self) -> bool:
        """True when the next step replays a captured step graph (this repository's engine only)."""
        return int(self.L.sph_app_step_graph_active(self.h)) == 1

    def body_pose(self, body: int) -> np.ndarray:
        """{cx, cy, cz, qx, qy, qz, qw} of one kinematic body."""
        out = np.zeros(7, np.float32)
        if self.L.sph_app_body_pose(self.h, C.c_int(body), out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_body_pose failed (reference engine or bad index)")
        return out

    def body_motion(self, body: int) -> np.ndarray:
        """{Vx, Vy, Vz, Ox, Oy, Oz} of one body (the integrated motion of a dynamic body)."""
        out = np.zeros(6, np.float32)
        if self.L.sph_app_body_motion(self.h, C.c_int(body), out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_body_motion failed (reference engine or bad index)")
        return out

    def body_impulse(self, body: int) -> np.ndarray:
        """{J, H} the fluid gave one body over the last step (two-way coupled systems; zero otherwise)."""
        out = np.zeros(6, np.float32)
        if self.L.sph_app_body_impulse(self.h, C.c_int(body), out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_body_impulse failed (reference engine or bad index)")
        return out

    def close(self):
        if getattr(self, "h", None):
            self.L.sph_app_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
