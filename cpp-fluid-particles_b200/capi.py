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
    "sphk_rheology_work_floats", "sphk_non_newtonian_viscosity", "sphk_non_newtonian_stats", "sphk_shear_rate", "sphk_rheology_eval",
    "sphk_visc_field_setup", "sphk_visc_field_matvec",
    "sphk_heat_substeps", "sphk_heat_step", "sphk_heat_conduction", "sphk_heat_stats", "sphk_thermal_viscosity",
    "sphk_thermal_viscosity_eval", "sphk_adhesion", "sphk_adhesion_accel", "sphk_adhesion_stats",
    "sphk_mesh_transform", "sphk_mesh_properties", "sphk_mesh_create", "sphk_mesh_destroy", "sphk_mesh_classify", "sphk_mesh_fill",
    "sphk_mesh_sample_surface", "sphk_probe_sample", "sphk_probe_lattice", "sphk_gauge_levels", "sphk_probe_series_create",
    "sphk_probe_series_destroy", "sphk_probes_record", "sphk_probe_series_read",
    "sphk_state_checksum_host", "sphk_state_crc32_host", "sphk_state_checksum_device", "sphk_checkpoint_save", "sphk_checkpoint_wait",
    "sphk_checkpoint_release", "sphk_state_open", "sphk_state_close", "sphk_state_section_bytes", "sphk_checkpoint_load",
    "sphk_checkpoint_invalidate", "sphk_tank_eval", "sphk_tank_accel_bound", "sphk_tank_set", "sphk_tank_force", "sphk_tank_time",
    "sphk_tank_set_time",
]
SPH_APP_FUNCTIONS = [
    "sph_app_create", "sph_app_destroy", "sph_app_step", "sph_app_fluid_size", "sph_app_boundary_size",
    "sph_app_download_fluid", "sph_app_download_boundary", "sph_app_upload_fluid", "sph_app_engine",
    "sph_app_submit", "sph_app_wait", "sph_app_dfsph_iterations", "sph_app_set_option", "sph_app_set_vorticity",
    "sph_app_create_with_bodies", "sph_app_set_body_motion", "sph_app_body_pose", "sph_app_step_graph_active",
    "sph_app_create_with_dynamic_bodies", "sph_app_body_motion", "sph_app_body_impulse", "sph_app_set_implicit_viscosity",
    "sph_app_viscosity_stats", "sph_app_create_open", "sph_app_open_boundary_stats", "sph_app_set_adaptive_dt", "sph_app_advance",
    "sph_app_adaptive_stats", "sph_app_set_rheology", "sph_app_rheology_stats", "sph_app_download_viscosity",
    "sph_app_set_thermal", "sph_app_set_thermal_viscosity", "sph_app_upload_temperature", "sph_app_download_temperature",
    "sph_app_thermal_stats", "sph_app_set_adhesion", "sph_app_adhesion_stats", "sph_app_load_obj", "sph_app_load_obj_error",
    "sph_app_set_probes", "sph_app_probe_series", "sph_app_sample_probes", "sph_app_sample_lattice",
    "sph_app_checkpoint", "sph_app_checkpoint_wait", "sph_app_restore", "sph_app_set_tank_motion", "sph_app_tank_state",
]

BODY_LIMIT = 64                      # SPHK_BODY_LIMIT
PROBE_FIELDS = 8                     # SPHK_PROBE_FIELDS: S, rho, vx, vy, vz, p, T, n
PROBE_LIMIT = 4096                   # SPHK_PROBE_LIMIT
GAUGE_LIMIT = 64                     # SPHK_GAUGE_LIMIT
GAUGE_MAX_SAMPLES = 1024             # SPHK_GAUGE_MAX_SAMPLES
PROBE_CAPACITY_LIMIT = 65536         # SPHK_PROBE_CAPACITY_LIMIT
THERMAL_GROUPS = 1 + BODY_LIMIT      # SPHK_THERMAL_GROUPS


class ThermalGroup(C.Structure):
    """sphk_thermal_group of sphk.h"""
    _fields_ = [("t", C.c_float), ("h", C.c_float)]


class Thermal(C.Structure):
    """sphk_thermal of sphk.h"""
    _fields_ = [("alpha", C.c_float), ("beta", C.c_float), ("t_ref", C.c_float), ("n_groups", C.c_int),
                ("groups", ThermalGroup * THERMAL_GROUPS)]


class ViscosityLaw(C.Structure):
    """sphk_viscosity_law of sphk.h"""
    _fields_ = [("nu_ref", C.c_float), ("e", C.c_float), ("t_ref", C.c_float), ("nu_min", C.c_float), ("nu_max", C.c_float)]


def thermal(spec: dict) -> Thermal:
    """sphk_thermal from dict(alpha, beta=0, t_ref=0, wall=(T, h) = (0, 0), bodies=[(T, h), ...], emitters=[T, ...]) (emitters is
    ignored here).  Unknown keys and more than BODY_LIMIT bodies raise ValueError; the ranges are checked by the library."""
    extra = set(spec) - {"alpha", "beta", "t_ref", "wall", "bodies", "emitters"}
    if extra:
        raise ValueError(f"unknown thermal keys {sorted(extra)}")
    bodies = list(spec.get("bodies", ()))
    if len(bodies) > BODY_LIMIT:
        raise ValueError(f"at most {BODY_LIMIT} bodies")
    t = Thermal()
    t.alpha, t.beta, t.t_ref = float(spec["alpha"]), float(spec.get("beta", 0.0)), float(spec.get("t_ref", 0.0))
    t.n_groups = 1 + len(bodies)
    for g, (T, h) in enumerate([tuple(spec.get("wall", (0.0, 0.0)))] + [tuple(b) for b in bodies]):
        t.groups[g].t, t.groups[g].h = float(T), float(h)
    return t


ADHESION_GROUPS = 1 + BODY_LIMIT     # SPHK_ADHESION_GROUPS


class Adhesion(C.Structure):
    """sphk_adhesion_setting of sphk.h"""
    _fields_ = [("n_groups", C.c_int), ("beta", C.c_float * ADHESION_GROUPS)]


TANK_HARMONICS = 4                   # SPHK_TANK_HARMONICS
TANK_STATE = 9                       # SPHK_TANK_STATE


class TankMotion(C.Structure):
    """sphk_tank_motion of sphk.h (sph_app_tank_motion has the same layout)"""
    _fields_ = [("axis", C.c_float * 3), ("pivot", C.c_float * 3), ("roll_amplitude", C.c_float), ("roll_omega", C.c_float),
                ("roll_phase", C.c_float), ("spin", C.c_float), ("accel", C.c_float * 3), ("n_harmonics", C.c_int),
                ("harmonic_amplitude", (C.c_float * 3) * TANK_HARMONICS), ("harmonic_omega", C.c_float * TANK_HARMONICS),
                ("harmonic_phase", C.c_float * TANK_HARMONICS), ("ramp", C.c_float)]


TANK_KEYS = {"axis", "pivot", "roll_amplitude", "roll_omega", "roll_phase", "spin", "accel", "harmonics", "ramp"}


def tank_motion(spec: dict) -> TankMotion:
    """sphk_tank_motion from dict(axis=(0, 0, 1), pivot=(0, 0, 0), roll_amplitude=0, roll_omega=0, roll_phase=0, spin=0,
    accel=(0, 0, 0), harmonics=[dict(amplitude=(ax, ay, az), omega=, phase=0), ...], ramp=0) (DESIGN.md section 2.15).  Unknown keys
    and more than TANK_HARMONICS harmonics raise ValueError; the ranges are checked by the library.  Unused entries are zero."""
    extra = set(spec) - TANK_KEYS
    if extra:
        raise ValueError(f"unknown tank keys {sorted(extra)}")
    harm = list(spec.get("harmonics", ()))
    if len(harm) > TANK_HARMONICS:
        raise ValueError(f"at most {TANK_HARMONICS} harmonics")
    m = TankMotion()
    m.axis[:] = [float(x) for x in spec.get("axis", (0.0, 0.0, 1.0))]
    m.pivot[:] = [float(x) for x in spec.get("pivot", (0.0, 0.0, 0.0))]
    m.roll_amplitude, m.roll_omega = float(spec.get("roll_amplitude", 0.0)), float(spec.get("roll_omega", 0.0))
    m.roll_phase, m.spin = float(spec.get("roll_phase", 0.0)), float(spec.get("spin", 0.0))
    m.accel[:] = [float(x) for x in spec.get("accel", (0.0, 0.0, 0.0))]
    m.n_harmonics = len(harm)
    for k, h in enumerate(harm):
        if set(h) - {"amplitude", "omega", "phase"}:
            raise ValueError(f"unknown harmonic keys {sorted(set(h) - {'amplitude', 'omega', 'phase'})}")
        m.harmonic_amplitude[k][:] = [float(x) for x in h.get("amplitude", (0.0, 0.0, 0.0))]
        m.harmonic_omega[k], m.harmonic_phase[k] = float(h.get("omega", 0.0)), float(h.get("phase", 0.0))
    m.ramp = float(spec.get("ramp", 0.0))
    return m


def adhesion(spec: dict) -> Adhesion:
    """sphk_adhesion_setting from dict(wall=beta, bodies=[beta, ...]).  Unknown keys and more than BODY_LIMIT bodies raise
    ValueError; the ranges are checked by the library."""
    extra = set(spec) - {"wall", "bodies"}
    if extra:
        raise ValueError(f"unknown adhesion keys {sorted(extra)}")
    bodies = [float(b) for b in spec.get("bodies", ())]
    if len(bodies) > BODY_LIMIT:
        raise ValueError(f"at most {BODY_LIMIT} bodies")
    a = Adhesion()
    a.n_groups = 1 + len(bodies)
    for g, beta in enumerate([float(spec.get("wall", 0.0))] + bodies):
        a.beta[g] = beta
    return a


# the solve's settings of a thermal viscosity dict, beside the law's own keys
THERMAL_VISCOSITY_DEFAULTS = {"nu_min": 0.0, "wall_factor": 0.0, "tol": 1e-4, "max_iter": 20}


def viscosity_law(spec: dict, t_ref: float) -> ViscosityLaw:
    """sphk_viscosity_law from dict(nu_ref, e, nu_max[, nu_min]) and the thermal setting's t_ref"""
    extra = set(spec) - {"nu_ref", "e", "nu_max"} - set(THERMAL_VISCOSITY_DEFAULTS)
    if extra:
        raise ValueError(f"unknown thermal viscosity keys {sorted(extra)}")
    v = ViscosityLaw()
    v.nu_ref, v.e, v.t_ref = float(spec["nu_ref"]), float(spec["e"]), float(t_ref)
    v.nu_min, v.nu_max = float(spec.get("nu_min", 0.0)), float(spec["nu_max"])
    return v

RHEOLOGY_CROSS, RHEOLOGY_HERSCHEL_BULKLEY = 1, 2   # SPHK_RHEOLOGY_* of sphk.h


class Rheology(C.Structure):
    """sphk_rheology of sphk.h"""
    _fields_ = [("model", C.c_int), ("params", C.c_float * 6), ("nu_min", C.c_float), ("nu_max", C.c_float)]


# the solve's settings of a rheology dict, beside the model's own keys
RHEOLOGY_SOLVE_DEFAULTS = {"beta": 0.0, "tol": 1e-4, "max_iter": 20}


def rheology(spec: dict) -> Rheology:
    """sphk_rheology from dict(model="cross", nu0, nu_inf, lam, m, nu_max[, nu_min]) or dict(model="hb", k, n, tau_y[, m_reg = 1000],
    nu_max[, nu_min]) (the solve's keys beta, tol and max_iter are ignored here).  Unknown models and keys raise ValueError; the
    ranges are checked by the library."""
    keys = {"cross": ("nu0", "nu_inf", "lam", "m"), "hb": ("k", "n", "tau_y", "m_reg")}
    model = spec.get("model")
    if model not in keys:
        raise ValueError(f"rheology model must be 'cross' or 'hb' (got {model!r})")
    extra = set(spec) - set(keys[model]) - {"model", "nu_min", "nu_max"} - set(RHEOLOGY_SOLVE_DEFAULTS)
    if extra:
        raise ValueError(f"unknown rheology keys {sorted(extra)}")
    r = Rheology()
    r.model = RHEOLOGY_CROSS if model == "cross" else RHEOLOGY_HERSCHEL_BULKLEY
    defaults = {"m_reg": 1000.0}
    for k, name in enumerate(keys[model]):
        if name not in spec and name not in defaults:
            raise ValueError(f"rheology {model!r} needs {name!r}")
        r.params[k] = float(spec.get(name, defaults.get(name, 0.0)))
    if "nu_max" not in spec:
        raise ValueError("rheology needs a finite nu_max")
    r.nu_min, r.nu_max = float(spec.get("nu_min", 0.0)), float(spec["nu_max"])
    return r


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


class SphkGauge(C.Structure):
    """sphk_gauge of sphk.h"""
    _fields_ = [("a", C.c_float * 3), ("b", C.c_float * 3), ("samples", C.c_int)]


def probe_points(points) -> np.ndarray:
    """(P, 3) float32 probe points; ValueError for a wrong shape, non-finite values or more than PROBE_LIMIT"""
    p = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
    if p.shape[0] > PROBE_LIMIT or not np.isfinite(p).all():
        raise ValueError(f"probes need finite (x, y, z) points, at most {PROBE_LIMIT}")
    return p


def gauge_structs(specs, threshold: float):
    """sphk_gauge[] from (a, b) or (a, b, k) tuples (k default 64); ValueError for a == b, k outside [2, GAUGE_MAX_SAMPLES],
    non-finite values, more than GAUGE_LIMIT gauges or a threshold that is not finite and > 0"""
    specs = list(specs)
    if len(specs) > GAUGE_LIMIT or not (np.isfinite(threshold) and threshold > 0):
        raise ValueError(f"at most {GAUGE_LIMIT} gauges and a finite threshold > 0")
    out = (SphkGauge * max(1, len(specs)))()
    for g, spec in zip(out, specs):
        a, b = np.asarray(spec[0], np.float32).reshape(3), np.asarray(spec[1], np.float32).reshape(3)
        k = int(spec[2]) if len(spec) > 2 else 64
        if not (np.isfinite(a).all() and np.isfinite(b).all()) or (a == b).all() or not 2 <= k <= GAUGE_MAX_SAMPLES:
            raise ValueError(f"a gauge needs finite a != b and 2 <= k <= {GAUGE_MAX_SAMPLES}: {spec}")
        g.a[:], g.b[:], g.samples = [float(x) for x in a], [float(x) for x in b], k
    return out, len(specs)


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
        L.sphk_rheology_work_floats.restype = C.c_longlong
        L.sphk_destroy.restype = None
        L.sphk_mg_destroy.restype = None
        L.sphk_mesh_destroy.restype = None
        L.sphk_probe_series_destroy.restype = None
        L.sphk_state_close.restype = None
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
        L.sph_app_load_obj_error.restype = C.c_char_p
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


class SphkStateConfig(C.Structure):
    """sphk_state_config (include/sphk.h): the configuration fingerprint of a checkpoint file."""
    _fields_ = [("solver", C.c_char * 16), ("capacity_fluid", C.c_int), ("capacity_boundary", C.c_int), ("n_boundary", C.c_int),
                ("n_bodies", C.c_int), ("cell_size", C.c_int * 3), ("flags", C.c_int), ("space_size", C.c_float * 3),
                ("cell_length", C.c_float), ("radius", C.c_float), ("dt", C.c_float), ("m0", C.c_float), ("rho0", C.c_float),
                ("rho_boundary", C.c_float), ("stiff", C.c_float), ("visc", C.c_float), ("surface_tension", C.c_float),
                ("air_pressure", C.c_float), ("gravity", C.c_float * 3), ("solver_args", C.c_float * 4),
                ("bodies_hash", C.c_ulonglong), ("open_hash", C.c_ulonglong), ("settings_hash", C.c_ulonglong)]


class SphkStateSection(C.Structure):
    """sphk_state_section (include/sphk.h): one named range of device (host = 0) or host (host = 1) memory."""
    _fields_ = [("name", C.c_char * 32), ("ptr", C.c_void_p), ("bytes", C.c_ulonglong), ("elem_size", C.c_uint), ("host", C.c_int)]


def state_hash(data: bytes) -> int:
    """sphk_state_checksum_host of host bytes"""
    buf = C.create_string_buffer(bytes(data), max(1, len(data)))
    h = C.c_ulonglong(0)
    check(sphk().sphk_state_checksum_host(buf, C.c_ulonglong(len(data)), C.byref(h)), "sphk_state_checksum_host")
    return int(h.value)


def state_user_bytes(path: str) -> int:
    """the size of a checkpoint file's user section (0 when the file cannot be read: the restore itself reports why)"""
    L = sphk()
    f, nb = C.c_void_p(), C.c_ulonglong(0)
    if L.sphk_state_open(os.fsencode(path), C.byref(f), None, C.c_int(0)):
        return 0
    try:
        return int(nb.value) if L.sphk_state_section_bytes(f, b"user", C.byref(nb)) == 0 else 0
    finally:
        L.sphk_state_close(f)


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

    def set_rheology(self, spec):
        """Non-Newtonian viscosity in every following step instead of the constant-nu solve (spec: a dict for capi.rheology plus
        beta, tol, max_iter; None: off).  Not on the reference engine."""
        if spec is None:
            rc = self.L.sph_app_set_rheology(self.h, C.c_int(0), None, C.c_float(0), C.c_float(0), C.c_float(0), C.c_float(0), C.c_int(0))
        else:
            r = rheology(spec)
            o = dict(RHEOLOGY_SOLVE_DEFAULTS, **{k: spec[k] for k in RHEOLOGY_SOLVE_DEFAULTS if k in spec})
            rc = self.L.sph_app_set_rheology(self.h, C.c_int(r.model), r.params, C.c_float(r.nu_min), C.c_float(r.nu_max),
                                             C.c_float(o["beta"]), C.c_float(o["tol"]), C.c_int(int(o["max_iter"])))
        if rc:
            raise RuntimeError("sph_app_set_rheology failed (reference engine or a refused setting)")

    def rheology_stats(self) -> dict:
        """of the last non-Newtonian solve: iterations, residual, gamma_max, nu_min, nu_max, at_nu_max"""
        it, res, g, lo, hi, k = C.c_int(0), C.c_float(0), C.c_float(0), C.c_float(0), C.c_float(0), C.c_int(0)
        if self.L.sph_app_rheology_stats(self.h, C.byref(it), C.byref(res), C.byref(g), C.byref(lo), C.byref(hi), C.byref(k)):
            raise RuntimeError("sph_app_rheology_stats failed (reference engine)")
        return {"iterations": it.value, "residual": res.value, "gamma_max": g.value, "nu_min": lo.value, "nu_max": hi.value,
                "at_nu_max": k.value}

    def download_viscosity(self) -> np.ndarray:
        """nu_i of the last non-Newtonian solve (float32[fluid size])"""
        out = np.zeros(int(self.L.sph_app_fluid_size(self.h)), np.float32)
        if self.L.sph_app_download_viscosity(self.h, out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_download_viscosity failed (reference engine)")
        return out

    def set_thermal(self, spec):
        """Heat transfer in every following step (spec: a dict for capi.thermal, with "emitters": [T, ...]; None: off).  Not on the
        reference engine."""
        if spec is None:
            rc = self.L.sph_app_set_thermal(self.h, C.c_int(0), *(C.c_float(0),) * 5, C.c_int(0), None, C.c_int(0), None)
        else:
            t = thermal(spec)
            bodies = np.ascontiguousarray(np.asarray(spec.get("bodies", []), np.float32).reshape(-1, 2))
            em = np.ascontiguousarray(np.asarray(spec.get("emitters", []), np.float32).reshape(-1))
            rc = self.L.sph_app_set_thermal(self.h, C.c_int(1), C.c_float(t.alpha), C.c_float(t.beta), C.c_float(t.t_ref),
                                            C.c_float(t.groups[0].t), C.c_float(t.groups[0].h), C.c_int(bodies.shape[0]),
                                            bodies.ctypes.data_as(C.c_void_p), C.c_int(em.size), em.ctypes.data_as(C.c_void_p))
        if rc:
            raise RuntimeError("sph_app_set_thermal failed (reference engine or a refused setting)")

    def set_thermal_viscosity(self, spec):
        """nu(T) instead of the constant-nu solve (spec: dict(nu_ref, e, nu_max, nu_min, wall_factor, tol, max_iter); None: off)"""
        if spec is None:
            rc = self.L.sph_app_set_thermal_viscosity(self.h, C.c_int(0), *(C.c_float(0),) * 6, C.c_int(0))
        else:
            v = viscosity_law(spec, 0.0)
            o = dict(THERMAL_VISCOSITY_DEFAULTS, **{k: spec[k] for k in THERMAL_VISCOSITY_DEFAULTS if k in spec})
            rc = self.L.sph_app_set_thermal_viscosity(self.h, C.c_int(1), C.c_float(v.nu_ref), C.c_float(v.e), C.c_float(v.nu_min),
                                                      C.c_float(v.nu_max), C.c_float(o["wall_factor"]), C.c_float(o["tol"]),
                                                      C.c_int(int(o["max_iter"])))
        if rc:
            raise RuntimeError("sph_app_set_thermal_viscosity failed (reference engine or a refused setting)")

    def upload_temperature(self, t):
        a = np.ascontiguousarray(t, np.float32)
        if a.size != int(self.L.sph_app_fluid_size(self.h)) or self.L.sph_app_upload_temperature(self.h, a.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_upload_temperature failed (reference engine or a wrong size)")

    def download_temperature(self) -> np.ndarray:
        out = np.zeros(int(self.L.sph_app_fluid_size(self.h)), np.float32)
        if self.L.sph_app_download_temperature(self.h, out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_download_temperature failed (reference engine)")
        return out

    def set_adhesion(self, spec):
        """Fluid-solid adhesion in every following step (spec: a dict for capi.adhesion; None: off).  Not on the reference engine."""
        if spec is None:
            rc = self.L.sph_app_set_adhesion(self.h, C.c_int(0), C.c_float(0), C.c_int(0), None)
        else:
            a = adhesion(spec)
            bodies = np.ascontiguousarray(np.asarray(spec.get("bodies", []), np.float32).reshape(-1))
            rc = self.L.sph_app_set_adhesion(self.h, C.c_int(1), C.c_float(a.beta[0]), C.c_int(bodies.size),
                                             bodies.ctypes.data_as(C.c_void_p))
        if rc:
            raise RuntimeError("sph_app_set_adhesion failed (reference engine or a refused setting)")

    def adhesion_stats(self) -> dict:
        """wetted particles and the largest |a_i| of the last step's adhesion sweep"""
        w, am = C.c_int(0), C.c_float(0)
        if self.L.sph_app_adhesion_stats(self.h, C.byref(w), C.byref(am)):
            raise RuntimeError("sph_app_adhesion_stats failed (reference engine)")
        return {"wetted": w.value, "max_accel": am.value}

    def set_tank_motion(self, spec):
        """Tank motion from the next step on (spec: a dict for capi.tank_motion; None: off).  Not on the reference engine."""
        rc = self.L.sph_app_set_tank_motion(self.h, None if spec is None else C.byref(tank_motion(spec)))
        if rc:
            raise RuntimeError("sph_app_set_tank_motion failed (reference engine or a refused setting)")

    def tank_state(self) -> dict:
        """the motion at the simulated time: {"t", "theta", "theta_dot", "theta_ddot", "accel" (a_w, world), "gravity" (R (G - a_w),
        tank axes)}"""
        t, v = C.c_double(0.0), (C.c_float * 9)()
        if self.L.sph_app_tank_state(self.h, C.byref(t), v):
            raise RuntimeError("sph_app_tank_state failed (reference engine)")
        return {"t": t.value, "theta": v[0], "theta_dot": v[1], "theta_ddot": v[2], "accel": np.array(v[3:6], np.float32),
                "gravity": np.array(v[6:9], np.float32)}

    def set_probes(self, points=(), gauges=(), threshold: float = 0.5, capacity: int = 1024):
        """Probes and water-level gauges recorded every following step (SPHSystem::setProbes; DESIGN.md section 2.13).  points: (P, 3);
        gauges: (a, b) or (a, b, k) tuples; no points and no gauges: off.  Not on the reference engine."""
        pts = probe_points(points)
        gs, ng = gauge_structs(gauges, threshold)
        ab = np.ascontiguousarray([[*g.a, *g.b] for g in gs[:ng]], np.float32).reshape(-1)
        k = np.ascontiguousarray([g.samples for g in gs[:ng]], np.int32)
        if self.L.sph_app_set_probes(self.h, C.c_int(pts.shape[0]), pts.ctypes.data_as(C.c_void_p), C.c_int(ng),
                                     ab.ctypes.data_as(C.c_void_p), k.ctypes.data_as(C.c_void_p), C.c_float(threshold), C.c_int(capacity)):
            raise RuntimeError("sph_app_set_probes failed (reference engine or a refused setting)")

    def probe_series(self) -> dict:
        """the recorded rows still in the ring, oldest first: steps (T,), times (T,), records (T, P, 8), levels (T, G), overwritten"""
        rows, npt, ng, over = C.c_int(0), C.c_int(0), C.c_int(0), C.c_longlong(0)
        if self.L.sph_app_probe_series(self.h, C.byref(rows), C.byref(npt), C.byref(ng), C.byref(over), None, None, None, None):
            raise RuntimeError("sph_app_probe_series failed (reference engine)")
        T, P, G = rows.value, npt.value, ng.value
        out = {"steps": np.zeros(T, np.int64), "times": np.zeros(T, np.float64), "records": np.zeros((T, P, PROBE_FIELDS), np.float32),
               "levels": np.zeros((T, G), np.float32), "overwritten": int(over.value)}
        if self.L.sph_app_probe_series(self.h, None, None, None, None, *[out[k].ctypes.data_as(C.c_void_p)
                                                                         for k in ("steps", "times", "records", "levels")]):
            raise RuntimeError("sph_app_probe_series failed")
        return out

    def sample_probes(self, points) -> np.ndarray:
        """records (P, 8) of the given points in the current state"""
        pts = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
        out = np.zeros((pts.shape[0], PROBE_FIELDS), np.float32)
        if self.L.sph_app_sample_probes(self.h, C.c_int(pts.shape[0]), pts.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_sample_probes failed (reference engine or a refused call)")
        return out

    def sample_lattice(self, origin, spacing: float, dims) -> np.ndarray:
        """records (nx, ny, nz, 8) of the lattice origin + spacing (i, j, k) in the current state"""
        o = np.ascontiguousarray(origin, np.float32)
        d = np.ascontiguousarray([int(x) for x in dims], np.int32)
        out = np.zeros((*[int(x) for x in d], PROBE_FIELDS), np.float32)
        if self.L.sph_app_sample_lattice(self.h, o.ctypes.data_as(C.c_void_p), C.c_float(spacing), d.ctypes.data_as(C.c_void_p),
                                         out.ctypes.data_as(C.c_void_p)):
            raise RuntimeError("sph_app_sample_lattice failed (reference engine or a refused call)")
        return out

    def checkpoint(self, path: str, user: bytes = b""):
        """Snapshot the state into `path` (SPHSystem::checkpoint; DESIGN.md section 2.14).  Returns once the snapshot is enqueued; the
        file is written behind the following steps (checkpoint_wait).  Not on the reference engine."""
        u = bytes(user)
        if self.L.sph_app_checkpoint(self.h, os.fsencode(path), u if u else None, C.c_int(len(u))):
            raise RuntimeError("sph_app_checkpoint refused (reference engine or a solver that does not describe its state)")

    def checkpoint_wait(self):
        """Wait for the last checkpoint's file; raises when it could not be written."""
        if self.L.sph_app_checkpoint_wait(self.h):
            raise RuntimeError("sph_app_checkpoint_wait: the checkpoint failed (see the printed message)")

    def restore(self, path: str) -> bytes:
        """Overwrite the state from a checkpoint of a system with the same configuration; returns the stored user bytes.  A refused
        restore (printed reason) changes nothing and raises."""
        nb = C.c_int(0)
        buf = C.create_string_buffer(max(1, state_user_bytes(path)))
        if self.L.sph_app_restore(self.h, os.fsencode(path), buf, C.c_int(len(buf)), C.byref(nb)):
            raise RuntimeError("sph_app_restore refused (see the printed message)")
        self.nF = self.fluid_count
        return buf.raw[:nb.value]

    def thermal_stats(self) -> dict:
        """substeps, max_courant, violators of the last step; t_min, t_max, heat (sum m T) now"""
        k, cmax, v, lo, hi, q = C.c_int(0), C.c_float(0), C.c_int(0), C.c_float(0), C.c_float(0), C.c_double(0)
        if self.L.sph_app_thermal_stats(self.h, C.byref(k), C.byref(cmax), C.byref(v), C.byref(lo), C.byref(hi), C.byref(q)):
            raise RuntimeError("sph_app_thermal_stats failed (reference engine)")
        return {"substeps": k.value, "max_courant": cmax.value, "violators": v.value, "t_min": lo.value, "t_max": hi.value,
                "heat": q.value}

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
