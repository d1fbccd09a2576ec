"""torch-tensor front end of the libsphk C-ABI (include/sphk.h).

PyTorch is used for device memory and streams only -- every kernel that runs is a libsphk kernel; there
is no torch arithmetic on the hot path and no CPU fallback.  `SphkSystem` mirrors the reference's
SPHSystem + solver step sequences (SPHSystem.cu:33-158, BasicSPHSolver.cu:237-260, DFSPHSolver.cu:33-72,
PBDSolver.cu:34-73) call for call, like cpp-fluid-particles_b200/host/sph_api.cpp does in C++; it exists
so that python drivers (tests, the multi-GPU slab driver) can interleave their own work (halo exchange)
between the C-ABI calls.
"""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np
import torch

from . import capi
from .capi import SphkGrid, SphkParticles, SphkScene, check

EPSILON = 1e-6


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def device_fluid_block(L, lattice, device, stream, j_begin: int = 0, j_count: int | None = None, capacity: int | None = None) -> torch.Tensor:
    """The fluid block of a device-side scene (sphk_scene_fluid_block): (capacity, 3) float32 tensor whose first
    ny * j_count * nz rows are the lattice columns [j_begin, j_begin + j_count) in the reference's push order."""
    (nx, ny, nz), origin = lattice
    j_count = nx - j_begin if j_count is None else j_count
    n = ny * j_count * nz
    out = torch.zeros((max(capacity or n, n, 1), 3), dtype=torch.float32, device=device)
    from .scene import SPACING
    check(L.sphk_scene_fluid_block(_ptr(out), C.c_int(nx), C.c_int(ny), C.c_int(nz), (C.c_float * 3)(*origin), C.c_float(float(SPACING)),
                                   C.c_int(j_begin), C.c_int(j_count), C.c_void_p(stream.cuda_stream)), "sphk_scene_fluid_block")
    return out


def device_boundary_shell(L, params, device, stream) -> torch.Tensor:
    """The six-face boundary shell of a device-side scene (sphk_scene_boundary_shell)."""
    cs = (C.c_int * 3)(*[int(c) for c in params.cell_size])
    n = int(L.sphk_scene_boundary_count(cs))
    out = torch.empty((n, 3), dtype=torch.float32, device=device)
    check(L.sphk_scene_boundary_shell(_ptr(out), cs, (C.c_float * 3)(*[float(x) for x in params.space]), C.c_void_p(stream.cuda_stream)),
          "sphk_scene_boundary_shell")
    return out


class ParticleSet:
    """Device arrays of one SPHParticles object (SPHParticles.h:56-59)."""

    def __init__(self, pos_host, device, capacity: int | None = None):
        """pos_host: (n, 3) host array, or a (n, 3) float32 tensor already on `device` (device-side scenes).  capacity (>= n):
        the arrays' length, of which the first n slots are live (open boundaries change n)."""
        n = pos_host.shape[0]
        self.n = n
        if isinstance(pos_host, torch.Tensor):
            self.pos = pos_host
        else:
            self.pos = torch.from_numpy(np.ascontiguousarray(pos_host, np.float32)).to(device)
        if capacity is not None and capacity > n:
            self.pos = torch.cat([self.pos, torch.zeros((capacity - n, 3), dtype=torch.float32, device=device)], 0).contiguous()
        n = self.pos.shape[0]
        self.vel = torch.zeros((n, 3), dtype=torch.float32, device=device)
        self.mass = torch.zeros(n, dtype=torch.float32, device=device)
        self.density = torch.zeros(n, dtype=torch.float32, device=device)
        self.pressure = torch.zeros(n, dtype=torch.float32, device=device)
        self.p2c = torch.zeros(n, dtype=torch.int32, device=device)

    def abi(self) -> SphkParticles:
        p = SphkParticles()
        p.pos, p.vel, p.mass = _ptr(self.pos), _ptr(self.vel), _ptr(self.mass)
        p.density, p.pressure, p.particle2cell = _ptr(self.density), _ptr(self.pressure), _ptr(self.p2c)
        p.n = self.n
        return p


class SphkOps:
    """The C-ABI calls and the three solver sequences over torch tensors.  Subclasses provide the tensors
    (fluid, boundary, cs_fluid, cs_boundary, solver buffers), ctx and params.  The sync_* hooks are no-ops on
    one GPU; the slab driver overrides them with halo exchanges."""

    list_capacity = 96               # SPHK_OPT_LIST_CAPACITY of ctx (set_option keeps it current)
    vorticity_eps = 0.0              # vorticity confinement strength (BasicSPHSolver::setVorticityConfinement); 0: off
    implicit_nu = 0.0                # implicit viscosity (BasicSPHSolver::setImplicitViscosity); 0: off
    _thermal = None
    _thermal_viscosity = None
    _rheology = None
    _adhesion = None
    _tank = None                     # tank motion (SPHSystem::setTankMotion): a capi.tank_motion dict; None: off
    heat_substeps = 0                # conduction substeps of the last step
    implicit_nu_boundary = 0.0
    implicit_tol = 1e-4
    implicit_max_iter = 20
    _step_dt = None                  # the dt of the step in flight (None: the scene's dt); CFL-adaptive systems set it per step
    pbd_last_dt = None               # PBD: the dt of the last predict (the interval the next projection acts on)
    _probe_series = None             # sphk_probe_series of set_probes (None: off)
    _probe_recorded = False          # the step in flight recorded a row
    steps_run = 0                    # steps run so far (the constructor's step is step 0)

    @property
    def dt(self) -> float:
        return self.p.dt if self._step_dt is None else self._step_dt

    # ---- multi-GPU hooks ---------------------------------------------------------------------------------
    def sync_vel(self):
        pass

    def sync_scalar(self, t):
        pass

    def sync_array(self, t):
        pass

    def sync_positions(self):
        pass

    def reduce_sum(self, x: float) -> float:
        return x

    def owned(self, t):
        """The slice of a per-particle tensor this rank owns (all of it on one GPU)."""
        return t

    def n_total(self) -> int:
        return self.fluid.n

    def _alloc_solver_buffers(self, n):
        dev = self.device
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)  # noqa: E731
        self.buffer3 = f(n, 3)          # BasicSPHSolver::bufferFloat3
        self.color_grad_buf = f(n, 3)   # second buffer: the fused viscosity+surface sweep needs deltaV and colour gradient at once
        self.fused = True               # fused sweeps (default, like the C++ class layer) or one kernel per launch site
        if self.solver == "dfsph":      # DFSPHSolver.h:58-62
            self.alpha, self.kappa, self.error, self.warm = f(n), f(n), f(n), f(n)
            self.max_iter = self.p.max_iter if self.p.max_iter > 0 else 20
            self.den_thr = self.p.density_error_threshold if self.p.max_iter > 0 else 1e-3
            self.div_thr = self.p.divergence_error_threshold if self.p.max_iter > 0 else 1e-3
        if self.solver == "pbd":        # PBDSolver.h:77-84
            self.pos_last, self.dpos, self.lam = f(n, 3), f(n, 3), f(n)
            self.pos_last_init = False
            self.max_iter = self.p.max_iter if self.p.max_iter > 0 else 20
            self.xsph_c, self.relaxation = 0.05, 0.75
        self.it_div = self.it_den = 0

    # ---- C-ABI plumbing ---------------------------------------------------------------------------
    def scene_abi(self) -> SphkScene:
        if self._scene is None:
            s = SphkScene()
            s.fluid, s.boundary = self.fluid.abi(), self.boundary.abi()
            s.cell_start_fluid, s.cell_start_boundary = _ptr(self.cs_fluid), _ptr(self.cs_boundary)
            s.radius = self.p.radius
            self._scene = s
        return self._scene

    def _s(self):
        return C.byref(self.scene_abi())

    def set_use_list(self, on: bool, skin_permille: int = 0):
        check(self.L.sphk_set_option(self.ctx, capi.OPT_NEIGHBOR_LIST, 1 if on else 0))
        check(self.L.sphk_set_option(self.ctx, capi.OPT_LIST_SKIN, int(skin_permille)))

    def build_neighbor_list(self):
        check(self.L.sphk_build_neighbor_list(self.ctx, self._s()), "sphk_build_neighbor_list")

    def search_boundary(self):
        p = self.boundary.abi()
        check(self.L.sphk_neighbor_search(self.ctx, 1, C.byref(p), _ptr(self.cs_boundary)), "sphk_neighbor_search(b)")

    # ---- kinematic bodies (DESIGN.md section 2.3) -------------------------------------------------------------------------
    n_bodies = 0

    def bodies_step(self):
        p = self.boundary.abi()
        check(self.L.sphk_bodies_step(self.ctx, C.byref(p), _ptr(self.cs_boundary), C.c_float(self.dt)), "sphk_bodies_step")

    def set_body_motion(self, body: int, linear_velocity, angular_velocity):
        """New motion of one body from the next step on (an asynchronous copy, like SPHSystem::setBodyMotion); the other
        bodies keep their device-side (for dynamic bodies: integrated) motion."""
        m = np.ascontiguousarray([*linear_velocity, *angular_velocity], np.float32)
        check(self.L.sphk_bodies_set_body_motion(self.ctx, C.c_int(body), m.ctypes.data_as(C.POINTER(C.c_float))),
              "sphk_bodies_set_body_motion")
        self.body_motion[body] = m
        if self.adaptive:            # the next step's dt must see the new motion, as SPHSystem::setBodyMotion
            self.measure_speed()

    # ---- two-way coupled bodies (DESIGN.md section 2.4) -----------------------------------------------------------------
    bodies_dynamic = False

    def bodies_react(self, c):
        """The bodies' reaction to the sweep just run (sphk_bodies_react); nothing without dynamic bodies."""
        if self.bodies_dynamic:
            check(self.L.sphk_bodies_react(self.ctx, self._s(), C.c_float(float(c))), "sphk_bodies_react")

    def bodies_integrate(self):
        if self.bodies_dynamic:
            check(self.L.sphk_bodies_integrate(self.ctx, C.c_float(self.dt), self._G), "sphk_bodies_integrate")

    def current_body_motion(self) -> np.ndarray:
        """(n_bodies, 6) motions {V, Omega} on the device (the integrated ones for dynamic bodies; the attribute body_motion
        is the host copy of the prescribed motions); synchronises."""
        out = np.zeros((self.n_bodies, 6), np.float32)
        check(self.L.sphk_bodies_get_motion(self.ctx, out.ctypes.data_as(C.POINTER(C.c_float))), "sphk_bodies_get_motion")
        return out

    def body_impulse(self) -> np.ndarray:
        """(n_bodies, 6) {J, H} the fluid gave each body over the last step (H about the body's centre; zero without dynamic
        bodies, as SPHSystem::getBodyImpulse); synchronises."""
        out = np.zeros((self.n_bodies, 6), np.float32)
        if not self.bodies_dynamic:
            return out
        check(self.L.sphk_bodies_get_impulse(self.ctx, out.ctypes.data_as(C.POINTER(C.c_float))), "sphk_bodies_get_impulse")
        return out

    def body_pose(self) -> np.ndarray:
        """(n_bodies, 7) poses {c, q = (x, y, z, w)}; synchronises."""
        out = np.zeros((self.n_bodies, 7), np.float32)
        check(self.L.sphk_bodies_get_pose(self.ctx, out.ctypes.data_as(C.POINTER(C.c_float))), "sphk_bodies_get_pose")
        return out

    def body_local(self) -> torch.Tensor:
        """(n_boundary, 4) carried {r_k, group} in the current boundary order (group 0: static, b + 1: body b)."""
        out = torch.zeros((self.boundary.n, 4), dtype=torch.float32, device=self.device)
        check(self.L.sphk_bodies_get_local(self.ctx, _ptr(out)), "sphk_bodies_get_local")
        return out

    def search_fluid(self):
        p = self.fluid.abi()
        check(self.L.sphk_neighbor_search(self.ctx, 0, C.byref(p), _ptr(self.cs_fluid)), "sphk_neighbor_search(f)")

    def boundary_mass(self):
        p = self.boundary.abi()
        check(self.L.sphk_boundary_mass(self.ctx, C.byref(p), _ptr(self.cs_boundary), C.c_float(self.p.rho_boundary),
                                        C.c_float(self.p.radius)), "sphk_boundary_mass")

    def permutation(self) -> torch.Tensor:
        out = torch.empty(self.fluid.n, dtype=torch.int32, device=self.device)
        check(self.L.sphk_get_permutation(self.ctx, _ptr(out), C.c_int(self.fluid.n)))
        return out

    def device_rcp(self, x: float) -> float:
        out = C.c_float()
        check(self.L.sphk_device_rcp(self.ctx, C.c_float(x), C.byref(out)))
        return float(out.value)

    def list_stats(self):
        out = (C.c_longlong * 3)()
        check(self.L.sphk_list_stats(self.ctx, self._s(), out))
        return {"max": int(out[0]), "overflow": int(out[1]), "total": int(out[2])}

    def neighbor_list(self):
        """(counts[n], entries[capacity/4, cap, 4]) of the current int32 list, as torch tensors."""
        n, cap, kmax = self.fluid.n, self.fluid.pos.shape[0], self.list_capacity
        cnt = torch.zeros(n, dtype=torch.int32, device=self.device)
        ent = torch.zeros(kmax * cap, dtype=torch.int32, device=self.device)
        check(self.L.sphk_get_neighbor_list(self.ctx, self._s(), _ptr(cnt), _ptr(ent)), "sphk_get_neighbor_list")
        return cnt, ent.view(kmax // 4, cap, 4)

    def tile_lists(self):
        """(counts[n], slots[ceil(capacity/8), cap, 8], windows[tiles, 18, 2]) of the current tile lists (SPHK_OPT_TILE = 1),
        as torch tensors; the slots are raw 16-bit values in an int16 tensor (read them as uint16)."""
        n, cap, kmax = self.fluid.n, self.fluid.pos.shape[0], self.list_capacity
        planes, tiles, wins = (kmax + 7) // 8, (n + capi.TILE_PARTICLES - 1) // capi.TILE_PARTICLES, capi.TILE_WINDOWS
        cnt = torch.zeros(n, dtype=torch.int32, device=self.device)
        slots = torch.zeros(planes * cap * 8, dtype=torch.int16, device=self.device)
        win = torch.zeros(tiles * wins * 2, dtype=torch.int32, device=self.device)
        check(self.L.sphk_get_tile_lists(self.ctx, self._s(), _ptr(cnt), _ptr(slots), _ptr(win)), "sphk_get_tile_lists")
        return cnt, slots.view(planes, cap, 8), win.view(tiles, wins, 2)

    def set_option(self, opt: int, value: int):
        check(self.L.sphk_set_option(self.ctx, int(opt), int(value)))
        if int(opt) == capi.OPT_LIST_CAPACITY:
            self.list_capacity = int(value)

    def export_dots(self):
        """generate_dots (vbo.cu:26-51): (dot, colour) device tensors for the fluid set."""
        n = self.fluid.n
        dot = torch.empty((n, 3), dtype=torch.float32, device=self.device)
        col = torch.empty((n, 3), dtype=torch.float32, device=self.device)
        p = self.fluid.abi()
        check(self.L.sphk_export_dots(self.ctx, C.byref(p), _ptr(dot), _ptr(col)), "sphk_export_dots")
        return dot, col

    def launch_count(self) -> int:
        return int(self.L.sphk_launch_count(self.ctx))

    def synchronize(self):
        check(self.L.sphk_synchronize(self.ctx))

    def refresh(self):
        check(self.L.sphk_refresh(self.ctx, self._s()))

    # ---- one entry per reference launch site --------------------------------------------------------
    def gravity(self):
        check(self.L.sphk_gravity(self.ctx, self._s(), C.c_float(self.dt), self._G), "sphk_gravity")

    def force(self):
        """BasicSPHSolver::force: the tank frame's body force while a motion is set, else gravity"""
        if self._tank is not None:
            self.tank_force()
        else:
            self.gravity()

    # ---- tank motion (no reference counterpart; DESIGN.md section 2.15) ------------------------------------------------------
    @property
    def tank(self):
        """the tank motion (a dict for capi.tank_motion) or None; setting it is SPHSystem::setTankMotion (the frame time starts at the
        simulated time), None is clearTankMotion.  ValueError for a setting the class layer refuses (the setting is kept)."""
        return self._tank

    @tank.setter
    def tank(self, spec):
        if spec is None:
            if self._tank is not None:
                check(self.L.sphk_tank_set(self.ctx, None, None), "sphk_tank_set")
            self._tank = None
        else:
            m = capi.tank_motion(spec)
            if self.L.sphk_tank_eval(C.byref(m), self._G, C.c_double(0.0), (C.c_float * capi.TANK_STATE)()) != 0:
                raise ValueError(f"tank motion refused: {spec}")
            if self._thermal is not None:
                raise ValueError("tank motion refused: not together with heat transfer")
            if (m.roll_amplitude != 0.0 or m.spin != 0.0) and getattr(self, "bodies_dynamic", False):
                raise ValueError("tank motion refused: a rotating tank with dynamic bodies")
            check(self.L.sphk_tank_set(self.ctx, C.byref(m), self._G), "sphk_tank_set")
            check(self.L.sphk_tank_set_time(self.ctx, C.c_double(self.simulated_time)), "sphk_tank_set_time")
            self._tank, self._tank_abi = dict(spec), m
        if getattr(self, "adaptive", False):
            self._rule.gravity = self._rule_gravity()

    def _rule_gravity(self) -> float:
        """the adaptive rule's |G|: |G|, or sphk_tank_accel_bound under a tank motion (as SPHSystem::ruleGravity)"""
        if self._tank is not None:
            b = C.c_double(0.0)
            check(self.L.sphk_tank_accel_bound(C.byref(self._tank_abi), self._G, self._space, C.byref(b)), "sphk_tank_accel_bound")
            return b.value
        g = [float(np.float32(x)) for x in self.p.gravity]
        return float(np.sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]))

    def tank_force(self, dt=None):
        """sphk_tank_force with the step's dt (or `dt`)"""
        check(self.L.sphk_tank_force(self.ctx, self._s(), C.c_float(self.dt if dt is None else dt)), "sphk_tank_force")

    def tank_state(self):
        """(device frame time, the last sphk_tank_force's state float[9] {theta, thd, thdd, R (G - a_w), a_w}); synchronises"""
        t, v = C.c_double(0.0), (C.c_float * capi.TANK_STATE)()
        check(self.L.sphk_tank_time(self.ctx, C.byref(t), v), "sphk_tank_time")
        return t.value, np.array(v[:], np.float32)

    def viscosity(self):
        check(self.L.sphk_viscosity(self.ctx, self._s(), _ptr(self.buffer3), C.c_float(self.p.rho0),
                                    C.c_float(self.p.visc), C.c_float(self.dt)), "sphk_viscosity")

    def color_grad(self):
        check(self.L.sphk_color_grad(self.ctx, self._s(), _ptr(self.buffer3), C.c_float(self.p.rho0),
                                     C.c_float(self.p.rho_boundary)), "sphk_color_grad")

    def surface(self):
        check(self.L.sphk_surface(self.ctx, self._s(), _ptr(self.buffer3), C.c_float(self.dt), C.c_float(self.p.rho0),
                                  C.c_float(self.p.surface_tension), C.c_float(self.p.air_pressure)), "sphk_surface")

    def density(self):
        check(self.L.sphk_density(self.ctx, self._s()), "sphk_density")

    def fused_density_color_grad(self, with_alpha: bool):
        if with_alpha:
            check(self.L.sphk_fused_dfsph_density_alpha_color_grad(self.ctx, self._s(), _ptr(self.alpha), _ptr(self.color_grad_buf),
                                                                   C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary)),
                  "sphk_fused_dfsph_density_alpha_color_grad")
        else:
            check(self.L.sphk_fused_density_color_grad(self.ctx, self._s(), _ptr(self.color_grad_buf), C.c_float(self.p.rho0),
                                                       C.c_float(self.p.rho_boundary)), "sphk_fused_density_color_grad")

    def fused_density_alpha_div_error(self, with_color_grad: bool):
        check(self.L.sphk_fused_dfsph_density_alpha_div_error(self.ctx, self._s(), _ptr(self.alpha),
                                                              _ptr(self.color_grad_buf) if with_color_grad else None,
                                                              C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary), _ptr(self.error),
                                                              _ptr(self.kappa), C.c_float(self.dt)),
              "sphk_fused_dfsph_density_alpha_div_error")

    def fused_viscosity_surface(self):
        check(self.L.sphk_fused_viscosity_surface(self.ctx, self._s(), _ptr(self.buffer3), _ptr(self.color_grad_buf),
                                                  C.c_float(self.p.rho0), C.c_float(self.p.visc), C.c_float(self.dt),
                                                  C.c_float(self.p.surface_tension), C.c_float(self.p.air_pressure)),
              "sphk_fused_viscosity_surface")

    # ---- vorticity confinement (no reference counterpart) ----------------------------------------------------------------
    def _vort_buffers(self):
        if getattr(self, "omega", None) is None:   # allocated on first use, like the class layer's
            n = self.buffer3.shape[0]
            self.omega = torch.zeros((n, 3), dtype=torch.float32, device=self.device)
            self.omega_norm = torch.zeros(n, dtype=torch.float32, device=self.device)
        return _ptr(self.omega), _ptr(self.omega_norm)

    def vorticity(self):
        check(self.L.sphk_vorticity(self.ctx, self._s(), *self._vort_buffers(), C.c_float(self.p.rho0)), "sphk_vorticity")

    def vorticity_confinement(self, eps=None):
        check(self.L.sphk_vorticity_confinement(self.ctx, self._s(), *self._vort_buffers(),
                                                C.c_float(self.vorticity_eps if eps is None else eps), C.c_float(self.dt),
                                                C.c_float(self.p.rho0)), "sphk_vorticity_confinement")

    def fused_viscosity_surface_vorticity(self):
        check(self.L.sphk_fused_viscosity_surface_vorticity(self.ctx, self._s(), _ptr(self.buffer3), _ptr(self.color_grad_buf),
                                                            C.c_float(self.p.rho0), C.c_float(self.p.visc), C.c_float(self.dt),
                                                            C.c_float(self.p.surface_tension), C.c_float(self.p.air_pressure),
                                                            *self._vort_buffers()), "sphk_fused_viscosity_surface_vorticity")

    def fused_pbd_xsph_vorticity(self, with_color_grad: bool):
        check(self.L.sphk_fused_pbd_xsph_vorticity(self.ctx, self._s(), C.c_float(self.xsph_c), C.c_float(self.p.rho0),
                                                   _ptr(self.buffer3) if with_color_grad else None, C.c_float(self.p.rho_boundary),
                                                   *self._vort_buffers()), "sphk_fused_pbd_xsph_vorticity")

    # ---- implicit viscosity (no reference counterpart; DESIGN.md section 2.5) --------------------------------------------
    def _visc_work(self):
        if getattr(self, "visc_work", None) is None:   # allocated on first use, like the class layer's
            n = self.buffer3.shape[0]
            self.visc_work = torch.zeros(int(self.L.sphk_implicit_viscosity_work_floats(C.c_int(n))), dtype=torch.float32,
                                         device=self.device)
        return _ptr(self.visc_work)

    def implicit_viscosity(self, nu=None, nu_boundary=None, tol=None, max_iter=None):
        """The implicit viscosity solve with the attributes' settings (or the arguments)."""
        a = lambda x, d: d if x is None else x  # noqa: E731
        check(self.L.sphk_implicit_viscosity(self.ctx, self._s(), self._visc_work(), C.c_float(a(nu, self.implicit_nu)),
                                             C.c_float(a(nu_boundary, self.implicit_nu_boundary)), C.c_float(self.dt),
                                             C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary),
                                             C.c_float(a(tol, self.implicit_tol)), C.c_int(int(a(max_iter, self.implicit_max_iter)))),
              "sphk_implicit_viscosity")

    def implicit_viscosity_stats(self):
        """(iterations, |r|_M / |b|_M) of the last solve; synchronises."""
        it, res = C.c_int(0), C.c_float(0.0)
        check(self.L.sphk_implicit_viscosity_stats(self.ctx, C.byref(it), C.byref(res)), "sphk_implicit_viscosity_stats")
        return int(it.value), float(res.value)

    def visc_implicit_setup(self, d_out, b_out, nu, nu_boundary):
        """D_i (n, 6) and b_i (n, 3) of the solve into the given tensors (one sweep)."""
        check(self.L.sphk_visc_implicit_setup(self.ctx, self._s(), _ptr(d_out), _ptr(b_out), C.c_float(nu), C.c_float(nu_boundary),
                                              C.c_float(self.dt), C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary)),
              "sphk_visc_implicit_setup")

    def visc_implicit_matvec(self, d_in, p_in, ap_out, nu):
        """(A p)_i (n, 3) from D (n, 6) and p (n, 3) (one sweep)."""
        check(self.L.sphk_visc_implicit_matvec(self.ctx, self._s(), _ptr(d_in), _ptr(p_in), _ptr(ap_out), C.c_float(nu),
                                               C.c_float(self.dt), C.c_float(self.p.rho0)), "sphk_visc_implicit_matvec")

    # ---- non-Newtonian viscosity (no reference counterpart; DESIGN.md section 2.9) ---------------------------------------
    def _rheo_buffers(self):
        if getattr(self, "rheo_work", None) is None:   # allocated on first use, like the class layer's
            n = self.buffer3.shape[0]
            self.rheo_work = torch.zeros(int(self.L.sphk_rheology_work_floats(C.c_int(n))), dtype=torch.float32, device=self.device)
            self.nu_field = torch.zeros(n, dtype=torch.float32, device=self.device)
        return _ptr(self.rheo_work), _ptr(self.nu_field)

    def non_newtonian_viscosity(self, spec=None):
        """The non-Newtonian viscosity solve with the `rheology` attribute's setting (or `spec`)."""
        spec = self.rheology if spec is None else spec
        r = capi.rheology(spec)
        o = dict(capi.RHEOLOGY_SOLVE_DEFAULTS, **{k: spec[k] for k in capi.RHEOLOGY_SOLVE_DEFAULTS if k in spec})
        work, nu = self._rheo_buffers()
        check(self.L.sphk_non_newtonian_viscosity(self.ctx, self._s(), work, nu, C.byref(r), C.c_float(o["beta"]), C.c_float(self.dt),
                                                  C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary), C.c_float(o["tol"]),
                                                  C.c_int(int(o["max_iter"]))), "sphk_non_newtonian_viscosity")

    def non_newtonian_stats(self) -> dict:
        """of the last solve (as capi.SphApp.rheology_stats); synchronises"""
        it, res, g, lo, hi, k = C.c_int(0), C.c_float(0), C.c_float(0), C.c_float(0), C.c_float(0), C.c_int(0)
        check(self.L.sphk_non_newtonian_stats(self.ctx, C.byref(it), C.byref(res), C.byref(g), C.byref(lo), C.byref(hi), C.byref(k)),
              "sphk_non_newtonian_stats")
        return {"iterations": it.value, "residual": res.value, "gamma_max": g.value, "nu_min": lo.value, "nu_max": hi.value,
                "at_nu_max": k.value}

    def shear_rate(self, gamma_out, nu_out, spec, grad_out=None, flag_out=None, beta=0.0):
        """gamma_dot (n), nu (n) and optionally grad v (n, 9) and the fallback flag (n, int32) of the shear sweep alone"""
        r = capi.rheology(spec)
        check(self.L.sphk_shear_rate(self.ctx, self._s(), _ptr(gamma_out), _ptr(nu_out), _ptr(grad_out) if grad_out is not None else None,
                                     _ptr(flag_out) if flag_out is not None else None, C.byref(r), C.c_float(beta),
                                     C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary)), "sphk_shear_rate")

    def rheology_eval(self, spec, gamma, nu_out):
        r = capi.rheology(spec)
        check(self.L.sphk_rheology_eval(self.ctx, C.byref(r), _ptr(gamma), _ptr(nu_out), C.c_int(gamma.numel())), "sphk_rheology_eval")

    def visc_field_setup(self, d_out, b_out, nu, beta):
        """D_i (n, 6) and b_i (n, 3) with the per-particle nu (n) (one mirror + one sweep)"""
        check(self.L.sphk_visc_field_setup(self.ctx, self._s(), _ptr(d_out), _ptr(b_out), _ptr(nu), C.c_float(beta), C.c_float(self.dt),
                                           C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary)), "sphk_visc_field_setup")

    def visc_field_matvec(self, d_in, p_in, ap_out, nu):
        check(self.L.sphk_visc_field_matvec(self.ctx, self._s(), _ptr(d_in), _ptr(p_in), _ptr(ap_out), _ptr(nu), C.c_float(self.dt),
                                            C.c_float(self.p.rho0)), "sphk_visc_field_matvec")

    # ---- heat transfer (no reference counterpart; DESIGN.md section 2.10) -------------------------------------------------
    @property
    def rheology(self):
        """non-Newtonian viscosity (BasicSPHSolver::setRheology): a dict for capi.rheology plus beta, tol, max_iter; replaces the
        implicit_nu solve.  None: off.  Refused (ValueError) while `thermal_viscosity` is set."""
        return self._rheology

    @rheology.setter
    def rheology(self, spec):
        if spec is not None and self._thermal_viscosity is not None:
            raise ValueError("a rheology is not supported together with a temperature-dependent viscosity")
        self._rheology = spec

    @property
    def thermal_viscosity(self):
        """temperature-dependent viscosity (BasicSPHSolver::setThermalViscosity): dict(nu_ref, e, nu_max, nu_min, wall_factor, tol,
        max_iter), solved instead of the implicit_nu solve while `thermal` is set.  Refused (ValueError) while `rheology` is set."""
        return self._thermal_viscosity

    @thermal_viscosity.setter
    def thermal_viscosity(self, spec):
        if spec is not None and self._rheology is not None:
            raise ValueError("a temperature-dependent viscosity is not supported together with a rheology")
        self._thermal_viscosity = spec

    @property
    def thermal(self):
        """heat transfer (BasicSPHSolver::setThermal): a dict for capi.thermal plus "emitters": [T, ...]; None: off.  The first
        setting allocates `temperature` (capacity-sized, the fluid's current order) filled with t_ref."""
        return self._thermal

    @thermal.setter
    def thermal(self, spec):
        if spec is not None:
            t = capi.thermal(spec)
            if len(spec.get("bodies", ())) > self.n_bodies:
                raise ValueError(f"{len(spec['bodies'])} body entries, but the system has {self.n_bodies} bodies")
            if self.L.sphk_heat_substeps(C.byref(t), C.c_float(self.p.radius), C.c_float(0.0), C.byref(C.c_int(0))):
                raise ValueError(f"thermal setting refused: {spec}")
            if self._tank is not None:
                raise ValueError("thermal setting refused: not under a tank motion (the buoyancy acts along the constant G)")
            if getattr(self, "temperature", None) is None:
                n = self.buffer3.shape[0]
                self.temperature = torch.full((n,), float(np.float32(t.t_ref)), dtype=torch.float32, device=self.device)
                self.heat_work = torch.zeros(n, dtype=torch.float32, device=self.device)
            self._thermal_abi = t
        self._thermal = spec

    def heat(self):
        """the heat stage of one step: sphk_heat_substeps, then that many sphk_heat_step"""
        k = C.c_int(1)
        check(self.L.sphk_heat_substeps(C.byref(self._thermal_abi), C.c_float(self.p.radius), C.c_float(self.dt), C.byref(k)),
              "sphk_heat_substeps")
        self.heat_substeps = k.value
        g = (C.c_float * 3)(*[float(x) for x in self.p.gravity])
        for j in range(k.value):
            check(self.L.sphk_heat_step(self.ctx, self._s(), C.byref(self._thermal_abi), _ptr(self.temperature), _ptr(self.heat_work),
                                        C.c_float(self.dt), C.c_int(j), C.c_int(k.value), C.c_float(self.p.rho0),
                                        C.c_float(self.p.rho_boundary), g), "sphk_heat_step")

    def heat_conduction(self, temperature, out, dt_sub=0.0, spec=None):
        """dT/dt (n) of the conduction sweep alone (and its statistics with dt_sub)"""
        t = capi.thermal(spec) if spec is not None else self._thermal_abi
        check(self.L.sphk_heat_conduction(self.ctx, self._s(), C.byref(t), _ptr(temperature), _ptr(out), C.c_float(dt_sub),
                                          C.c_float(self.p.rho0), C.c_float(self.p.rho_boundary)), "sphk_heat_conduction")

    def thermal_stats(self) -> dict:
        """as capi.SphApp.thermal_stats; synchronises"""
        cmax, v, lo, hi, q = C.c_float(0), C.c_int(0), C.c_float(0), C.c_float(0), C.c_double(0)
        t = getattr(self, "temperature", None)
        n = self.fluid.n if t is not None else 0
        check(self.L.sphk_heat_stats(self.ctx, _ptr(t) if n else None, _ptr(self.fluid.mass) if n else None, C.c_int(n), C.byref(cmax), C.byref(v),
                                     C.byref(lo), C.byref(hi), C.byref(q)), "sphk_heat_stats")
        return {"substeps": self.heat_substeps, "max_courant": cmax.value, "violators": v.value, "t_min": lo.value, "t_max": hi.value,
                "heat": q.value}

    def _thermal_law(self, spec=None):
        spec = self.thermal_viscosity if spec is None else spec
        o = dict(capi.THERMAL_VISCOSITY_DEFAULTS, **{k: spec[k] for k in capi.THERMAL_VISCOSITY_DEFAULTS if k in spec})
        return capi.viscosity_law(spec, self._thermal_abi.t_ref), o

    def thermal_viscosity_solve(self):
        """the nu(T) solve with the `thermal_viscosity` setting, from the current temperatures"""
        law, o = self._thermal_law()
        if getattr(self, "nu_field", None) is None:
            self.nu_field = torch.zeros(self.buffer3.shape[0], dtype=torch.float32, device=self.device)
        work, nu = self._visc_work(), _ptr(self.nu_field)
        check(self.L.sphk_thermal_viscosity(self.ctx, self._s(), work, nu, _ptr(self.temperature), C.byref(law),
                                            C.c_float(o["wall_factor"]), C.c_float(self.dt), C.c_float(self.p.rho0),
                                            C.c_float(self.p.rho_boundary), C.c_float(o["tol"]), C.c_int(int(o["max_iter"]))),
              "sphk_thermal_viscosity")

    # ---- fluid-solid adhesion (no reference counterpart; DESIGN.md section 2.11) -------------------------------------------
    @property
    def adhesion(self):
        """fluid-solid adhesion (BasicSPHSolver::setAdhesion): dict(wall=beta, bodies=[beta, ...]) for capi.adhesion; None: off.
        More body entries than the system has bodies, and values the library refuses, raise ValueError."""
        return self._adhesion

    @adhesion.setter
    def adhesion(self, spec):
        if spec is not None:
            a = capi.adhesion(spec)
            if len(spec.get("bodies", ())) > self.n_bodies:
                raise ValueError(f"{len(spec['bodies'])} body entries, but the system has {self.n_bodies} bodies")
            if not all(np.isfinite(a.beta[g]) and a.beta[g] >= 0.0 for g in range(a.n_groups)):
                raise ValueError(f"adhesion setting refused: {spec}")
            self._adhesion_abi = a
        self._adhesion = spec

    def adhesion_step(self):
        """v += dt a_i with the `adhesion` setting (and the reaction on dynamic bodies)"""
        check(self.L.sphk_adhesion(self.ctx, self._s(), C.byref(self._adhesion_abi), C.c_float(self.dt), C.c_float(self.p.rho0),
                                   C.c_float(self.p.rho_boundary)), "sphk_adhesion")

    def adhesion_accel(self, out, spec=None):
        """a_i (n, 3) of the adhesion sweep alone, with `spec` or the current setting"""
        a = capi.adhesion(spec) if spec is not None else self._adhesion_abi
        check(self.L.sphk_adhesion_accel(self.ctx, self._s(), C.byref(a), _ptr(out), C.c_float(self.p.rho0),
                                         C.c_float(self.p.rho_boundary)), "sphk_adhesion_accel")

    def adhesion_stats(self) -> dict:
        """as capi.SphApp.adhesion_stats; synchronises"""
        w, am = C.c_int(0), C.c_float(0)
        check(self.L.sphk_adhesion_stats(self.ctx, C.byref(w), C.byref(am)), "sphk_adhesion_stats")
        return {"wetted": w.value, "max_accel": am.value}

    # ---- probes and water-level gauges (no reference counterpart; DESIGN.md section 2.13) ----------------------------------
    def _probe_sources(self):
        """the pressure of a WCSPH step (DFSPH and PBD keep none) and the temperatures while heat transfer is on, as pointers"""
        p = _ptr(self.fluid.pressure) if self.solver not in ("dfsph", "pbd") else None
        t = _ptr(self.temperature) if self._thermal is not None else None
        return p, t

    def probe_sample(self, points: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
        """records (P, 8) {S, rho, vx, vy, vz, p, T, n} of the device points (P, 3) in the current state (sphk_probe_sample)"""
        points = points.contiguous()
        out = torch.empty((points.shape[0], capi.PROBE_FIELDS), dtype=torch.float32, device=self.device) if out is None else out
        check(self.L.sphk_probe_sample(self.ctx, self._s(), _ptr(points), C.c_int(points.shape[0]), *self._probe_sources(), _ptr(out)),
              "sphk_probe_sample")
        return out

    def probe_lattice(self, origin, spacing: float, dims, out: torch.Tensor | None = None) -> torch.Tensor:
        """records (nx, ny, nz, 8) of the lattice origin + spacing (i, j, k), z fastest (sphk_probe_lattice)"""
        d = [int(x) for x in dims]
        out = torch.empty((*d, capi.PROBE_FIELDS), dtype=torch.float32, device=self.device) if out is None else out
        o = (C.c_float * 3)(*[float(x) for x in origin])
        check(self.L.sphk_probe_lattice(self.ctx, self._s(), o, C.c_float(spacing), (C.c_int * 3)(*d), *self._probe_sources(), _ptr(out)),
              "sphk_probe_lattice")
        return out

    def gauge_levels(self, gauges, threshold: float = 0.5, out: torch.Tensor | None = None) -> torch.Tensor:
        """levels (G,) of (a, b[, k]) gauges in the current state (sphk_gauge_levels)"""
        gs, ng = capi.gauge_structs(gauges, threshold)
        out = torch.empty(ng, dtype=torch.float32, device=self.device) if out is None else out
        check(self.L.sphk_gauge_levels(self.ctx, self._s(), gs, C.c_int(ng), C.c_float(threshold), _ptr(out)), "sphk_gauge_levels")
        return out

    def thermal_viscosity_eval(self, spec, t_ref, temperature, nu_out):
        law = capi.viscosity_law(spec, t_ref)
        check(self.L.sphk_thermal_viscosity_eval(self.ctx, C.byref(law), _ptr(temperature), _ptr(nu_out), C.c_int(temperature.numel())),
              "sphk_thermal_viscosity_eval")

    def pressure(self):
        check(self.L.sphk_pressure(self.ctx, self._s(), C.c_float(self.p.rho0), C.c_float(self.p.stiff)), "sphk_pressure")

    def pressure_force(self):
        check(self.L.sphk_pressure_force(self.ctx, self._s(), C.c_float(self.dt)), "sphk_pressure_force")

    def advect(self):
        check(self.L.sphk_advect(self.ctx, self._s(), C.c_float(self.dt), self._space), "sphk_advect")

    def dfsph_density_alpha(self):
        check(self.L.sphk_dfsph_density_alpha(self.ctx, self._s(), _ptr(self.alpha)), "sphk_dfsph_density_alpha")

    def dfsph_div_error(self):
        check(self.L.sphk_dfsph_div_error(self.ctx, self._s(), _ptr(self.alpha), _ptr(self.error), _ptr(self.kappa),
                                          C.c_float(self.dt), C.c_float(self.p.rho0)), "sphk_dfsph_div_error")

    def dfsph_div_correct(self, stiff=None):
        check(self.L.sphk_dfsph_div_correct(self.ctx, self._s(), _ptr(self.kappa if stiff is None else stiff)),
              "sphk_dfsph_div_correct")

    def dfsph_den_error(self, accumulate_warm: bool):
        check(self.L.sphk_dfsph_den_error(self.ctx, self._s(), _ptr(self.alpha), _ptr(self.error), _ptr(self.kappa),
                                          C.c_float(self.dt), C.c_float(self.p.rho0),
                                          _ptr(self.warm) if accumulate_warm else None), "sphk_dfsph_den_error")

    def dfsph_den_correct(self, stiff=None):
        check(self.L.sphk_dfsph_den_correct(self.ctx, self._s(), _ptr(self.kappa if stiff is None else stiff),
                                            C.c_float(self.dt)), "sphk_dfsph_den_correct")

    def reduce_abs_sum(self, x: torch.Tensor) -> float:
        out = C.c_float()
        check(self.L.sphk_reduce_abs_sum(self.ctx, _ptr(x), C.c_int(x.numel()), C.byref(out)))
        return float(out.value)

    def permute(self, arr: torch.Tensor, width: int):
        check(self.L.sphk_permute(self.ctx, _ptr(arr), C.c_int(width), C.c_int(self.fluid.n)), "sphk_permute")

    def copy(self, dst: torch.Tensor, src: torch.Tensor):
        check(self.L.sphk_copy(self.ctx, _ptr(dst), _ptr(src), C.c_int(src.numel())), "sphk_copy")

    def pbd_density_lambda(self):
        check(self.L.sphk_pbd_density_lambda(self.ctx, self._s(), _ptr(self.lam), C.c_float(self.p.rho0),
                                             C.c_float(self.relaxation)), "sphk_pbd_density_lambda")

    def pbd_delta_pos_apply(self):
        check(self.L.sphk_pbd_delta_pos_apply(self.ctx, self._s(), _ptr(self.lam), _ptr(self.dpos),
                                              C.c_float(self.p.rho0), self._space), "sphk_pbd_delta_pos_apply")

    def pbd_dt_prev(self) -> float:
        """the dt of the last predict (the step's own dt before the first), as PBDSolver::historyTimeStep"""
        return self.dt if self.pbd_last_dt is None else self.pbd_last_dt

    def pbd_velocity_from_positions(self):
        check(self.L.sphk_pbd_velocity_from_positions(self.ctx, self._s(), _ptr(self.pos_last), C.c_float(self.pbd_dt_prev())),
              "sphk_pbd_velocity_from_positions")

    def fused_pbd_xsph_color_grad(self):
        check(self.L.sphk_fused_pbd_xsph_color_grad(self.ctx, self._s(), C.c_float(self.xsph_c), C.c_float(self.p.rho0), _ptr(self.buffer3),
                                                    C.c_float(self.p.rho_boundary)), "sphk_fused_pbd_xsph_color_grad")

    def pbd_xsph(self):
        check(self.L.sphk_pbd_xsph(self.ctx, self._s(), C.c_float(self.xsph_c), C.c_float(self.p.rho0)), "sphk_pbd_xsph")

    # ---- solver sequences ----------------------------------------------------------------------------
    def _surface_enabled(self) -> bool:
        return self.p.surface_tension > EPSILON or self.p.air_pressure > EPSILON

    def _run(self, op, sync=None, tensor=None, split=True):
        """One sweep followed by the halo refresh of what it produced (`sync`: None | "vel" | "scalar" | "array").
        On one GPU the refresh is a no-op; the slab driver overrides this to overlap the exchange with the sweep
        (split=False: the sweep reads the field it writes -- Jacobi velocity updates -- and must run in one piece)."""
        op()
        if sync == "vel":
            self.sync_vel()
        elif sync == "scalar":
            self.sync_scalar(tensor)
        elif sync == "array":
            self.sync_array(tensor)

    def _velocity_stage(self, xsph: bool = False):
        """The velocity terms of every solver's step, in the class layer's order (BasicSPHSolver::velocityStage): vorticity omega,
        viscosity (xsph: PBD's XSPH), surface tension, adhesion, implicit viscosity, vorticity confinement, heat.  With fused sweeps and not xsph
        the colour gradient must be in color_grad_buf already (the density sweep computes it)."""
        surface, vort = self._surface_enabled(), self.vorticity_eps > 0
        if vort:
            self._vort_buffers()
        if self.fused and xsph and (surface or vort):
            # XSPH + colour gradient (positions are final after the projection) + omega from the velocities XSPH reads
            if vort:
                self._run(lambda: self.fused_pbd_xsph_vorticity(surface), "vel", split=False)
                self.sync_scalar(self.omega_norm)
            else:
                self._run(self.fused_pbd_xsph_color_grad, "vel", split=False)
            if surface:
                self.sync_array(self.buffer3)
                self._run(self.surface, "vel")
        elif self.fused and not xsph and surface:
            # viscosity + surface (+ omega from the velocities the viscosity term reads)
            if vort:
                self._run(self.fused_viscosity_surface_vorticity, "scalar", self.omega_norm, split=False)
                self.sync_vel()
            else:
                self._run(self.fused_viscosity_surface, "vel", split=False)
        else:
            if vort:
                self._run(self.vorticity, "scalar", self.omega_norm)
            self._run(self.pbd_xsph if xsph else self.viscosity, "vel", split=False)
            if surface:              # handleSurface, BasicSPHSolver.cu:262-275
                self._run(self.color_grad, "array", self.buffer3)
                self._run(self.surface, "vel")
        if self.adhesion is not None:
            self._run(self.adhesion_step, "vel")
        if self.rheology is not None:       # replaces the constant-nu solve
            self._run(self.non_newtonian_viscosity, "vel")
        elif self.thermal is not None and self.thermal_viscosity is not None:
            self._run(self.thermal_viscosity_solve, "vel")
        elif self.implicit_nu > 0:
            self._run(self.implicit_viscosity, "vel")
        if vort:
            self._run(self.vorticity_confinement, "vel")
        if self.thermal is not None:
            self._run(self.heat, "vel")

    def _carry_temperature(self):
        """the temperatures follow their particles through this step's search (BasicSPHSolver::beginStep)"""
        if self.thermal is not None:
            self.permute(self.temperature, 1)

    def step_wcsph(self):            # BasicSPHSolver.cu:237-260
        self.set_use_list(self.use_list)
        self._carry_temperature()
        self.force()
        if self.fused:               # density (+ colour gradient) before the velocity terms: it reads positions and masses only
            if self._surface_enabled():
                self._run(lambda: self.fused_density_color_grad(False), "array", self.color_grad_buf)
            else:
                self.density()
        self._velocity_stage()
        if not self.fused:
            self.density()
        self.pressure()
        self.sync_array(self.fluid.density); self.sync_array(self.fluid.pressure)
        self.pressure_force()
        self.bodies_react(-np.float32(self.dt))
        self.advect()

    def step_dfsph(self):            # DFSPHSolver.cu:33-72
        self.set_use_list(self.use_list)
        self._carry_temperature()
        n, rho0 = self.n_total(), self.p.rho0
        if self.fused:               # density/alpha (+ colour gradient) + the first divergence error (:341) in one sweep
            surface = self._surface_enabled()
            self._run(lambda: self.fused_density_alpha_div_error(surface), "scalar", self.kappa)
            if surface:
                self.sync_array(self.color_grad_buf)
        else:
            self.dfsph_density_alpha()
            self._run(self.dfsph_div_error, "scalar", self.kappa)
        total, it = 3.4e38, 0        # correctDivergenceError :331-363
        while (it < 1 or total > self.div_thr * n * rho0) and it < self.max_iter:
            self._run(self.dfsph_div_correct, "vel")
            self.bodies_react(1.0)
            it += 1
            if it == self.max_iter:  # the loop ends whatever the error is, and nothing reads it again: dead sweep
                break
            self._run(self.dfsph_div_error, "scalar", self.kappa)
            if self.div_thr >= 0:    # negative threshold: the test cannot depend on the sum (Q11) -> no host sync
                total = self.reduce_sum(self.reduce_abs_sum(self.owned(self.error)))
        self.it_div = it
        self.force()
        self._velocity_stage()
        total, it = 3.4e38, 0        # project :160-210
        self.permute(self.warm, 1)
        self._run(lambda: self.dfsph_den_correct(self.warm), "vel")
        inv_dt = np.float32(1.0) / np.float32(self.dt)
        self.bodies_react(inv_dt)
        self._run(lambda: self.dfsph_den_error(False), "scalar", self.kappa)
        self.copy(self.warm, self.kappa)
        while (it < 2 or total > self.den_thr * n * rho0) and it < self.max_iter:
            self._run(self.dfsph_den_correct, "vel")
            self.bodies_react(inv_dt)
            self._run(lambda: self.dfsph_den_error(True), "scalar", self.kappa)
            it += 1
            if it >= 2 and self.den_thr >= 0:
                total = self.reduce_sum(self.reduce_abs_sum(self.owned(self.error)))
        self.it_den = it
        self.advect()

    def step_pbd(self) -> bool:      # PBDSolver.cu:34-73; returns False for the "throwing" first call (Q6)
        if not self.pos_last_init:
            self.copy(self.pos_last, self.fluid.pos)
            self.pos_last_init = True
            return False
        self.set_use_list(self.use_list, 150 if self.use_list else 0)   # skin list: positions move inside the step
        self._carry_temperature()
        self.permute(self.pos_last, 3)
        c = np.float32(1.0) / (np.float32(self.p.rho0) * np.float32(self.pbd_dt_prev()))
        for _ in range(self.max_iter):
            self._run(self.pbd_density_lambda, "scalar", self.lam)
            self.bodies_react(c)     # before the positions move: the pairs of this correction
            self.pbd_delta_pos_apply(); self.sync_positions()
        self.pbd_velocity_from_positions()
        self._velocity_stage(xsph=True)
        self.force()
        self.copy(self.pos_last, self.fluid.pos)
        self.advect()
        self.pbd_last_dt = self.dt
        return True

    # ---- open boundaries (DESIGN.md section 2.6) --------------------------------------------------------------------------
    open = False

    def _set_live(self, n: int):
        self.fluid.n = n
        self._scene = None           # the cached scene carries the count

    def _history(self):
        """(history tensor, kind) of the solver for sphk_emit: DFSPH warm start (1: zero), PBD last position (2: x - dt v)"""
        if self.solver == "dfsph":
            return self.warm, 1
        if self.solver == "pbd":
            return self.pos_last, 2
        return None, 0

    def open_emit(self) -> int:
        """sinks over the live slots, then every emitter's scheduled layers into the slots after them (as SPHSystem::openEmit);
        returns the emitted count"""
        n, cap = self.fluid.n, self.fluid.pos.shape[0]
        p = self.fluid.abi()
        if self._sinks.shape[0]:
            check(self.L.sphk_sinks_apply(self.ctx, C.byref(p), self._sinks.ctypes.data_as(C.POINTER(C.c_float)),
                                          C.c_int(self._sinks.shape[0])), "sphk_sinks_apply")
        hist, kind = self._history()
        hist_dt = self.pbd_dt_prev() if self.solver == "pbd" else self.dt
        e = 0
        for k, em in enumerate(self._emitters):
            per = em.width * em.height
            fit = min((cap - n - e) // per, 65536)
            off = (C.c_float * max(fit, 1))()
            carry, sched = C.c_double(self.emitter_carry[k]), C.c_int(0)
            check(self.L.sphk_emitter_advance(C.byref(em), C.byref(carry), C.c_float(self.dt), C.c_int(fit), off, C.byref(sched)),
                  "sphk_emitter_advance")
            self.emitter_carry[k] = carry.value
            layers = min(sched.value, fit)
            self._open_stats["refused"] += (sched.value - layers) * per
            if layers == 0:
                continue
            check(self.L.sphk_emit(self.ctx, C.byref(p), C.c_int(n + e), C.byref(em), C.c_int(layers), off, C.c_float(self.p.m0),
                                   C.c_float(hist_dt), _ptr(hist), C.c_int(kind)), "sphk_emit")
            if self.thermal is not None:     # the emitter's temperature (default t_ref) into its new slots
                ts = self.thermal.get("emitters", [])
                check(self.L.sphk_fill(self.ctx, _ptr(self.temperature[n + e:]), C.c_int(layers * per),
                                       C.c_float(ts[k] if k < len(ts) else self._thermal_abi.t_ref)), "sphk_fill")
            e += layers * per
            self._open_stats["emitted"] += layers * per
        return e

    def open_set_count(self, searched: int) -> int:
        """after the search of `searched` slots: L = searched - removed, sphk_fluid_set_count(L)"""
        removed = C.c_int(0)
        if self._sinks.shape[0]:
            check(self.L.sphk_sinks_removed(self.ctx, C.byref(removed)), "sphk_sinks_removed")
        live = searched - removed.value
        check(self.L.sphk_fluid_set_count(self.ctx, _ptr(self.cs_fluid), C.c_int(live)), "sphk_fluid_set_count")
        self._set_live(live)
        self._open_stats["removed"] += removed.value
        return live

    @property
    def fluid_count(self) -> int:
        return self.fluid.n

    def open_boundary_stats(self) -> dict:
        """cumulative {"emitted", "removed", "refused"} particle counts"""
        return dict(self._open_stats)

    def open_check(self) -> int:
        """sticky bits of the per-step count check (sphk_open_check; 0 = fine); synchronises"""
        bits = C.c_int(0)
        check(self.L.sphk_open_check(self.ctx, C.byref(bits)), "sphk_open_check")
        return int(bits.value)

    # ---- CFL-adaptive time stepping (DESIGN.md section 2.8): the same C rule and order as SPHSystem ------------------------------
    adaptive = False
    last_dt = None                   # the dt of the last step (float32 value)
    simulated_time = 0.0             # the double sum of the float dt of every step

    def set_adaptive(self, C_: float, dt_min: float = 0.0, dt_max: float = 0.0):
        """SPHSystem::setAdaptiveTimeStep: from the next step on, every step runs at the rule's dt (0 = the defaults: dt_max = the
        scene's dt, dt_min = dt_max / 64).  Raises ValueError for values the rule refuses (the setting is kept)."""
        f = lambda x: float(np.float32(x))  # noqa: E731
        r = capi.SphkTimeStepRule()
        r.cfl = f(C_)
        r.dt_max = f(dt_max) if dt_max > 0 else f(self.p.dt)
        r.dt_min = f(dt_min) if dt_min > 0 else float(np.float32(r.dt_max) / np.float32(64.0))
        r.radius = f(self.p.radius)
        r.gravity = self._rule_gravity()
        dt, flags = C.c_float(0.0), C.c_int(0)
        if not (dt_min >= 0 and dt_max >= 0) or self.L.sphk_time_step(C.byref(r), C.c_double(0.0), C.c_double(0.0), C.c_double(0.0),
                                                                      C.byref(dt), C.byref(flags)) != 0:
            raise ValueError(f"adaptive time stepping needs C > 0, dt_min >= 0 and dt_max >= 0 (finite) with dt_min <= dt_max "
                             f"(got {C_}, {dt_min}, {dt_max})")
        if self._emitters and r.dt_max > f(self.p.dt):
            raise ValueError(f"dt_max {dt_max} is above the scene's dt {self.p.dt}, for which the emitters' layers were placed")
        self._rule = r
        self.adaptive = True
        self.adaptive_stats = {"speed": 0.0, "source": 0, "min_clamps": 0, "nonfinite_steps": 0, "frame_min_dt": 0.0}
        self.measure_speed()

    def disable_adaptive(self):
        self.adaptive = False
        self._step_dt = None

    def measure_speed(self):
        """enqueues the speed bound of the current state (sphk_step_speed)"""
        p = self.fluid.abi()
        check(self.L.sphk_step_speed(self.ctx, C.byref(p), C.c_int(1 if self.n_bodies else 0)), "sphk_step_speed")

    def refresh_speed_bound(self):
        """SPHSystem::refreshSpeedBound: measure the bound again after writing velocities or positions between steps"""
        if self.adaptive:
            self.measure_speed()

    def speed_result(self):
        """((fluid max |v|, body max |V| + |Omega| r_max), non-finite count) of the last measure_speed"""
        v, bad = (C.c_float * 2)(), C.c_int(0)
        check(self.L.sphk_step_speed_result(self.ctx, v, C.byref(bad)), "sphk_step_speed_result")
        return (float(v[0]), float(v[1])), int(bad.value)

    def choose_time_step(self, remaining: float):
        """(dt, frame_end) of the next step, as SPHSystem::chooseTimeStep"""
        (vf, vb), bad = self.speed_result()
        vmax, source = vf, 0
        if vb > vmax:
            vmax, source = vb, 1
        for em in self._emitters:
            if em.speed > vmax:
                vmax, source = float(em.speed), 2
        dt, flags = C.c_float(0.0), C.c_int(0)
        check(self.L.sphk_time_step(C.byref(self._rule), C.c_double(vmax), C.c_double(self.last_dt), C.c_double(remaining),
                                    C.byref(dt), C.byref(flags)), "sphk_time_step")
        st = self.adaptive_stats
        st["speed"], st["source"] = vmax, source
        st["min_clamps"] += bool(flags.value & capi.DT_MIN_CLAMP)
        st["nonfinite_steps"] += bool(flags.value & capi.DT_NONFINITE) or bad > 0
        return float(dt.value), bool(flags.value & capi.DT_FRAME_END)

    def advance(self, frame_seconds: float) -> int:
        """SPHSystem::advance: CFL substeps until frame_seconds of simulated time have passed; returns their count"""
        if not self.adaptive or not (frame_seconds > 0) or not np.isfinite(frame_seconds):
            raise ValueError("advance needs an adaptive system and a finite frame > 0")
        elapsed, k, end, min_dt = 0.0, 0, False, np.inf
        while not end:
            dt, end = self.choose_time_step(frame_seconds - elapsed)
            self._run_step(dt)
            elapsed += dt
            min_dt = min(min_dt, dt)
            k += 1
        self.adaptive_stats["frame_min_dt"] = min_dt
        return k

    def step(self):                  # SPHSystem.cu:129-158 (no host sync here, except for the speed bound of an adaptive system)
        self._run_step(self.choose_time_step(0.0)[0] if self.adaptive else float(np.float32(self.p.dt)))

    def _run_step(self, dt: float):
        self._step_dt = dt if self.adaptive else None
        self._probe_recorded = False
        if self._step_body() is not False and self.adaptive:
            self.measure_speed()     # after the step's last velocity write
        self.last_dt = dt
        self.simulated_time += dt
        if self._probe_recorded:     # the row's step index and simulated time, kept on the host beside the device ring
            self._probe_meta[self._probe_rows % len(self._probe_meta)] = (self.steps_run, self.simulated_time)
            self._probe_rows += 1
        self.steps_run += 1

    def set_probes(self, points=(), gauges=(), threshold: float = 0.5, capacity: int = 1024):
        """probes (P, 3) and (a, b[, k]) gauges recorded into a device ring of `capacity` rows at the end of every following step
        (SPHSystem::setProbes); no points and no gauges: off.  ValueError for a setting the library refuses (the setting is kept)."""
        pts = capi.probe_points(points)
        gs, ng = capi.gauge_structs(gauges, threshold)
        if pts.shape[0] == 0 and ng == 0:
            self._close_probes()
            return
        series = C.c_void_p()
        rc = self.L.sphk_probe_series_create(C.byref(series), pts.ctypes.data_as(C.c_void_p), C.c_int(pts.shape[0]), gs, C.c_int(ng),
                                             C.c_float(threshold), C.c_int(int(capacity)), C.c_void_p(self.stream.cuda_stream))
        if rc:
            raise ValueError(f"probe setting refused: {capi.sphk().sphk_error_string(C.c_int(rc)).decode()}")
        self._close_probes()
        self._probe_series, self._probe_shape = series, (pts.shape[0], ng, int(capacity))
        self._probe_meta, self._probe_rows = [(0, 0.0)] * int(capacity), 0

    def _close_probes(self):
        if self._probe_series:
            self.L.sphk_probe_series_destroy(self._probe_series)
            self._probe_series = None

    def probe_series(self) -> dict:
        """as capi.SphApp.probe_series; synchronises"""
        if not self._probe_series:
            return None
        P, G, cap = self._probe_shape
        rec, lev = np.zeros((cap, P, capi.PROBE_FIELDS), np.float32), np.zeros((cap, G), np.float32)
        count, rows = C.c_longlong(0), C.c_int(0)
        check(self.L.sphk_probe_series_read(self._probe_series, C.byref(count), C.c_int(cap), rec.ctypes.data_as(C.c_void_p),
                                            lev.ctypes.data_as(C.c_void_p), C.byref(rows)), "sphk_probe_series_read")
        T, n = rows.value, count.value
        meta = [self._probe_meta[r % cap] for r in range(n - T, n)]
        return {"steps": np.array([m[0] for m in meta], np.int64), "times": np.array([m[1] for m in meta], np.float64),
                "records": rec[:T], "levels": lev[:T], "overwritten": n - T}

    def _step_body(self):
        e = self.open_emit() if self.open else 0
        if self.n_bodies:            # bodies move before the fluid search, as in SPHSystem::step
            self.bodies_step()
        if self.open:
            self._set_live(self.fluid.n + e)
            if self.fluid.n == 0:
                return
        self.search_fluid()
        if self.open and self.open_set_count(self.fluid.n) == 0:
            return
        if self.use_list:            # (the C++ layer builds the list lazily in the first sweep; same kernel)
            self.set_use_list(True, 150 if self.solver == "pbd" else 0)
            self.build_neighbor_list()
        if not self._step_solver():
            return False             # the "throwing" first call: no sweep ran, nothing to integrate (as in SPHSystem::step)
        self.bodies_integrate()
        if self._probe_series:       # as SPHSystem::recordProbes, after the bodies' integration
            check(self.L.sphk_probes_record(self.ctx, self._s(), self._probe_series, *self._probe_sources()), "sphk_probes_record")
            self._probe_recorded = True

    def _step_solver(self) -> bool:
        """the solver's part of a step; False for PBD's "throwing" first call"""
        if self.solver == "dfsph":
            self.step_dfsph()
        elif self.solver == "pbd":
            return self.step_pbd()
        else:
            self.step_wcsph()
        return True

    def state(self) -> dict:
        """the live fluid particles (and every boundary particle) on the host"""
        self.synchronize()
        g = lambda t: t.detach().cpu().numpy()  # noqa: E731
        n = self.fluid.n
        return {"pos": g(self.fluid.pos[:n]), "vel": g(self.fluid.vel[:n]), "density": g(self.fluid.density[:n]),
                "pressure": g(self.fluid.pressure[:n]), "mass": g(self.fluid.mass[:n]), "p2c": g(self.fluid.p2c[:n]),
                "cell_start": g(self.cs_fluid), "posB": g(self.boundary.pos), "massB": g(self.boundary.mass),
                "p2cB": g(self.boundary.p2c), "cell_startB": g(self.cs_boundary)}

    def close(self):
        self._close_probes()
        if self.ctx:
            self.L.sphk_synchronize(self.ctx)
            self.L.sphk_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SphkSystem(SphkOps):
    """SPHSystem + solver over the C-ABI with torch tensors.  construct(step0=True) reproduces the
    reference constructor including its implicit first step (Q3)."""

    def __init__(self, scene, device="cuda:0", use_list: bool | None = None, list_capacity: int | None = None,
                 step0: bool = True, bodies=None, max_fluid: int | None = None, emitters=None, sinks=None, adaptive=None, tank=None):
        """emitters / sinks: open boundaries (DESIGN.md section 2.6), the same C entries in the same order as SPHSystem::step.
        emitters: dicts {"origin", "direction", "speed", "spacing", "width", "height"} (sphk_emitter); sinks: (lo, hi) boxes; max_fluid:
        the capacity of the fluid set (default: the initial count).  fluid_count is the live count.
        bodies: rigid bodies (DESIGN.md sections 2.3, 2.4), a list of dicts with "points" (k, 3) body coordinates,
        "position" (3,), "orientation" (x, y, z, w) unit quaternion, "linear_velocity" (3,), "angular_velocity" (3,) in the
        world frame, and optionally "mass" (> 0: dynamic, two-way coupled; default 0: kinematic, and held -- its reaction reported --
        when another body is dynamic) and "inertia" (3,) principal
        moments about the centre in the axes of "points".  Masses are in the fluid's units, m0 / spacing^3 per unit volume
        (not rho0).  Their particles follow the static boundary set; every step() moves them before the fluid search.
        adaptive: dict(C=, dt_min=0, dt_max=0): CFL-adaptive time stepping (set_adaptive) from the step after the constructor's on.
        tank: a tank motion (the `tank` property; DESIGN.md section 2.15) from the step after the constructor's on."""
        self.L = capi.sphk()
        self.p = scene.params
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.stream = torch.cuda.current_stream(self.device)
        if scene.fluid is None:      # device-side scene (SURVEY 8f-4): no host particle arrays
            self.fluid = ParticleSet(device_fluid_block(self.L, scene.lattice, self.device, self.stream), self.device)
            self.boundary = ParticleSet(device_boundary_shell(self.L, self.p, self.device, self.stream), self.device)
        else:
            self.fluid = ParticleSet(scene.fluid, self.device, max_fluid)
            self.boundary = ParticleSet(scene.boundary, self.device)
        if scene.fluid is None and max_fluid is not None:
            self.fluid = ParticleSet(self.fluid.pos, self.device, max_fluid)
        self._emitters = [capi.emitter_struct(e) for e in (emitters or [])]
        self._sinks = capi.sink_boxes(sinks or [])
        if len(self._emitters) > capi.MAX_EMITTERS or self._sinks.shape[0] > capi.MAX_SINKS:
            raise ValueError("at most 16 emitters and 16 sinks")
        for em in self._emitters:          # the library's validation (sphk_emitter_axes)
            check(self.L.sphk_emitter_axes(C.byref(em), (C.c_float * 9)()), "sphk_emitter_axes")
        if (self._sinks.shape[0] and not (self._sinks[:, :3] < self._sinks[:, 3:]).all()) or not np.isfinite(self._sinks).all():
            raise ValueError("a sink needs finite lo < hi on every axis")
        self.open = bool(self._emitters) or self._sinks.shape[0] > 0
        self.emitter_carry = [0.0] * len(self._emitters)
        self._open_stats = {"emitted": 0, "removed": 0, "refused": 0}
        bodies = list(bodies or [])
        self.n_bodies = len(bodies)
        if bodies:                   # static set + the bodies' particles (placed by the first boundary search)
            n_static = self.boundary.n
            pts = [np.asarray(b["points"], np.float32).reshape(-1, 3) for b in bodies]
            local = torch.from_numpy(np.concatenate(pts, 0)).to(self.device)
            self.boundary = ParticleSet(torch.cat([self.boundary.pos, local], 0).contiguous(), self.device)
            begin = np.concatenate([[0], np.cumsum([len(q) for q in pts])]) + n_static
            self._body_begin = (C.c_int * (self.n_bodies + 1))(*[int(x) for x in begin])
            self._body_local = np.ascontiguousarray(local.cpu().numpy())
            self._body_pose = np.array([[*b["position"], *b["orientation"]] for b in bodies], np.float32)
            self.body_motion = np.array([[*b["linear_velocity"], *b["angular_velocity"]] for b in bodies], np.float32)
        nc = self.p.ncells
        self.cs_fluid = torch.zeros(nc + 1, dtype=torch.int32, device=self.device)
        self.cs_boundary = torch.zeros(nc + 1, dtype=torch.int32, device=self.device)
        g = SphkGrid()
        g.cell_size[:] = [int(c) for c in self.p.cell_size]
        g.cell_length = self.p.cell_length
        self.ctx = C.c_void_p()
        check(self.L.sphk_create(C.byref(self.ctx), C.c_int(self.fluid.pos.shape[0]), C.c_int(self.boundary.n), C.byref(g),
                                 C.c_void_p(self.stream.cuda_stream)), "sphk_create")
        if list_capacity is not None:
            self.set_option(capi.OPT_LIST_CAPACITY, list_capacity)
        self.solver = self.p.solver
        self.last_dt = float(np.float32(self.p.dt))   # as SPHSystem's _lastDt: the dt_prev of a first adaptive step
        self.use_list = True if use_list is None else bool(use_list)
        n = self.fluid.n
        self._alloc_solver_buffers(self.fluid.pos.shape[0])
        self._scene = None
        self._G = (C.c_float * 3)(*[float(x) for x in self.p.gravity])
        self._space = (C.c_float * 3)(*[float(x) for x in self.p.space])
        if self.n_bodies:
            p = self.boundary.abi()
            fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
            check(self.L.sphk_bodies_init(self.ctx, C.byref(p), C.c_int(int(self._body_begin[0])), C.c_int(self.n_bodies),
                                          self._body_begin, fp(self._body_local), fp(self._body_pose), fp(self.body_motion)),
                  "sphk_bodies_init")
            mi = capi.body_mass_inertia(bodies)
            self._body_mi = mi
            if (mi[:, 0] > 0).any():     # as SPHSystem: held bodies (mass 0) then report their reaction too
                check(self.L.sphk_bodies_set_dynamics(self.ctx, fp(mi), self._space), "sphk_bodies_set_dynamics")
                self.bodies_dynamic = True
        # SPHSystem.cu:68-76 (with bodies the boundary search also places them at their initial pose)
        self.search_boundary()
        self.boundary_mass()
        check(self.L.sphk_fill(self.ctx, _ptr(self.fluid.mass), C.c_int(n), C.c_float(self.p.m0)), "sphk_fill")
        self.search_fluid()
        if step0:
            self.step()
        if adaptive is not None:
            self.set_adaptive(adaptive["C"], adaptive.get("dt_min", 0.0), adaptive.get("dt_max", 0.0))
        if tank is not None:
            self.tank = tank

    # ---- checkpoints (DESIGN.md section 2.14): the class layer's sections, names and config record ---------------------------------
    _STATE_RECORD = struct.Struct("<6qd4f2i")          # SPHSystem::StateRecord

    def _state_config(self) -> capi.SphkStateConfig:
        f32 = lambda x: float(np.float32(x))  # noqa: E731
        c = capi.SphkStateConfig()
        p = self.p
        c.solver = {"wcsph": b"wcsph", "dfsph": b"dfsph", "pbd": b"pbd"}[self.solver]
        c.capacity_fluid, c.capacity_boundary = self.fluid.pos.shape[0], self.boundary.n
        c.n_boundary, c.n_bodies = self.boundary.n, self.n_bodies
        c.cell_size[:] = [int(x) for x in p.cell_size]
        c.flags = (1 if self.fused else 0) | (2 if self.solver == "dfsph" else 0) | (4 if self.open else 0) | \
            (8 if self.bodies_dynamic else 0) | (16 if getattr(self, "adaptive", False) else 0)
        c.space_size[:] = [f32(x) for x in p.space]
        c.cell_length, c.radius, c.dt, c.m0, c.rho0 = p.cell_length, p.radius, p.dt, p.m0, p.rho0
        c.rho_boundary, c.stiff, c.visc, c.surface_tension, c.air_pressure = p.rho_boundary, p.stiff, p.visc, p.surface_tension, p.air_pressure
        c.gravity[:] = [f32(x) for x in p.gravity]
        if self.solver == "dfsph":
            c.solver_args[:] = [self.den_thr, self.div_thr, float(self.max_iter), 0.0]
        elif self.solver == "pbd":
            c.solver_args[:] = [float(self.max_iter), self.xsph_c, self.relaxation, 0.0]
        M = (1 << 64) - 1
        if self.n_bodies:
            local = np.ascontiguousarray(self._body_local, np.float32).tobytes()
            mi = np.ascontiguousarray(self._body_mi, np.float32).tobytes()
            c.bodies_hash = (capi.state_hash(local) * 31 + capi.state_hash(mi) + int(self._body_begin[0])) & M
        if self.open:
            em = b"".join(bytes(e) for e in self._emitters)
            c.open_hash = (capi.state_hash(em) * 31 + capi.state_hash(self._sinks.astype(np.float32).tobytes()) + len(self._emitters)) & M
        f, i, b = (lambda x: struct.pack("<f", x)), (lambda x: struct.pack("<i", int(x))), (lambda x: struct.pack("<?", bool(x)))
        st = f(self.vorticity_eps)
        if self.implicit_nu > 0.0:
            st += f(self.implicit_nu) + f(self.implicit_nu_boundary) + f(self.implicit_tol) + i(self.implicit_max_iter)
        st += b(self._rheology is not None)
        if self._rheology is not None:
            o = dict(capi.RHEOLOGY_SOLVE_DEFAULTS, **{k: self._rheology[k] for k in capi.RHEOLOGY_SOLVE_DEFAULTS if k in self._rheology})
            st += bytes(capi.rheology(self._rheology)) + f(o["beta"]) + f(o["tol"]) + i(o["max_iter"])
        st += b(self._thermal is not None)
        if self._thermal is not None:
            st += bytes(self._thermal_abi) + b"".join(f(t) for t in self._thermal.get("emitters", ()))
            st += b(self._thermal_viscosity is not None)
            if self._thermal_viscosity is not None:
                v = capi.viscosity_law(self._thermal_viscosity, 0.0)
                o = dict(capi.THERMAL_VISCOSITY_DEFAULTS, **{k: self._thermal_viscosity[k] for k in capi.THERMAL_VISCOSITY_DEFAULTS
                                                             if k in self._thermal_viscosity})
                st += f(v.nu_ref) + f(v.e) + f(v.nu_min) + f(v.nu_max) + f(o["wall_factor"]) + f(o["tol"]) + i(o["max_iter"])
        st += b(self._adhesion is not None)
        if self._adhesion is not None:
            st += bytes(self._adhesion_abi)
        if getattr(self, "adaptive", False):
            st += bytes(self._rule)
        if self._tank is not None:
            st += bytes(self._tank_abi)
        c.settings_hash = (capi.state_hash(st) + len(st)) & M
        return c

    def _state_sections(self, n: int, rec, carry, motion, user):
        """the class layer's sections in its order (SPHSystem::stateSections); host sections point at the given ctypes buffers"""
        out = []

        def add(name, ptr, nbytes, elem, host=False):
            s = capi.SphkStateSection()
            s.name, s.ptr, s.bytes, s.elem_size, s.host = name.encode(), ptr, nbytes, elem, int(host)
            out.append(s)
        fl, bd = self.fluid, self.boundary
        add("fluid.pos", _ptr(fl.pos), 12 * n, 12)
        add("fluid.vel", _ptr(fl.vel), 12 * n, 12)
        add("fluid.mass", _ptr(fl.mass), 4 * n, 4)
        add("fluid.density", _ptr(fl.density), 4 * n, 4)
        add("fluid.pressure", _ptr(fl.pressure), 4 * n, 4)
        add("fluid.particle2cell", _ptr(fl.p2c), 4 * n, 4)
        add("boundary.pos", _ptr(bd.pos), 12 * bd.n, 12)
        add("boundary.mass", _ptr(bd.mass), 4 * bd.n, 4)
        if self._thermal is not None:
            add("solver.temperature", _ptr(self.temperature), 4 * n, 4)
            add("solver.temperature_set", C.addressof(self._state_tset), 1, 1, True)
        if self.solver == "dfsph":
            add("solver.dfsph_warm_stiffness", _ptr(self.warm), 4 * n, 4)
        if self.solver == "pbd":
            add("solver.pbd_pos_last", _ptr(self.pos_last), 12 * n, 12)
            add("solver.pbd_last_predict_dt", C.addressof(self._state_pdt), 4, 4, True)
            add("solver.pbd_pos_last_initialized", C.addressof(self._state_pinit), 1, 1, True)
        add("system.record", C.addressof(rec), len(rec), 8, True)
        if self.open:
            add("system.emitter_carry", C.addressof(carry), C.sizeof(carry), 8, True)
        if self.n_bodies:
            add("system.body_motion", C.addressof(motion), C.sizeof(motion), 4, True)
        add("user", C.addressof(user) if len(user) else None, len(user), 1, True)
        return (capi.SphkStateSection * max(1, len(out)))(*out), len(out)

    def save_state(self, path: str, user: bytes = b""):
        """SPHSystem::checkpoint: the same library entries, sections and config record, so the file restores in any layer.  Returns
        once the snapshot is enqueued; wait_state() waits for the file."""
        n = self.fluid.n
        st = getattr(self, "adaptive_stats", None) or {"speed": 0.0, "source": 0, "min_clamps": 0, "nonfinite_steps": 0, "frame_min_dt": 0.0}
        o = self._open_stats
        rec = C.create_string_buffer(self._STATE_RECORD.pack(
            self.steps_run, o["emitted"], o["removed"], o["refused"], st["min_clamps"], st["nonfinite_steps"], self.simulated_time,
            self.last_dt, self.dt, st["speed"], st["frame_min_dt"], st["source"], n), self._STATE_RECORD.size)
        carry = (C.c_double * max(1, len(self.emitter_carry)))(*self.emitter_carry)
        motion = (C.c_float * max(1, 6 * self.n_bodies))(*(np.asarray(self.body_motion, np.float32).reshape(-1) if self.n_bodies else [0.0]))
        u = C.create_string_buffer(bytes(user), max(1, len(user)))
        self._state_tset = C.c_bool(self._thermal is not None)
        self._state_pdt = C.c_float(self.pbd_last_dt or 0.0)
        self._state_pinit = C.c_bool(bool(getattr(self, "pos_last_init", False)))
        secs, k = self._state_sections(n, rec, carry, motion, u if len(user) else b"")
        cfg = self._state_config()
        check(self.L.sphk_checkpoint_save(self.ctx, os.fsencode(path), C.byref(cfg), secs, C.c_int(k)), "sphk_checkpoint_save")

    def wait_state(self):
        """SPHSystem::waitCheckpoint: raises RuntimeError with the library's message when the file could not be written"""
        msg = C.create_string_buffer(512)
        if self.L.sphk_checkpoint_wait(self.ctx, msg, C.c_int(512)):
            raise RuntimeError(f"checkpoint failed: {msg.value.decode()}")

    def load_state(self, path: str) -> bytes:
        """SPHSystem::restore: overwrites the state from a file of any layer (same configuration); returns the user bytes.  A refused
        load changes nothing and raises RuntimeError naming the field or section at fault."""
        msg = C.create_string_buffer(512)
        self.L.sphk_checkpoint_wait(self.ctx, msg, C.c_int(512))
        f = C.c_void_p()
        if self.L.sphk_state_open(os.fsencode(path), C.byref(f), msg, C.c_int(512)):
            raise RuntimeError(f"restore refused: {msg.value.decode()}")
        try:
            pos_b, user_b = C.c_ulonglong(0), C.c_ulonglong(0)
            if self.L.sphk_state_section_bytes(f, b"fluid.pos", C.byref(pos_b)) or self.L.sphk_state_section_bytes(f, b"user", C.byref(user_b)):
                raise RuntimeError("restore refused: the file has no fluid.pos or user section")
            n = self.fluid.n
            if self.open:
                if pos_b.value % 12 or pos_b.value // 12 > self.fluid.pos.shape[0]:
                    raise RuntimeError(f"restore refused: section 'fluid.pos' holds {pos_b.value} bytes, more than the capacity")
                n = pos_b.value // 12
            rec = C.create_string_buffer(self._STATE_RECORD.size)
            carry = (C.c_double * max(1, len(self.emitter_carry)))()
            motion = (C.c_float * max(1, 6 * self.n_bodies))()
            u = C.create_string_buffer(max(1, user_b.value))
            self._state_tset, self._state_pdt, self._state_pinit = C.c_bool(False), C.c_float(0.0), C.c_bool(False)
            secs, k = self._state_sections(n, rec, carry, motion, u if user_b.value else b"")
            cfg = self._state_config()
            if self.L.sphk_checkpoint_load(self.ctx, f, C.byref(cfg), secs, C.c_int(k), msg, C.c_int(512)):
                raise RuntimeError(f"restore refused: {msg.value.decode()}")
        finally:
            self.L.sphk_state_close(f)
        (self.steps_run, e, r, x, mc, nf, self.simulated_time, last_dt, step_dt, speed, fmin, src, _live) = self._STATE_RECORD.unpack(rec.raw)
        self.last_dt = last_dt
        if self.open:
            self._set_live(n)
            self._open_stats = {"emitted": e, "removed": r, "refused": x}
            self.emitter_carry = list(carry)[:len(self.emitter_carry)]
        if getattr(self, "adaptive", False):
            self.adaptive_stats = {"speed": speed, "source": src, "min_clamps": mc, "nonfinite_steps": nf, "frame_min_dt": fmin}
        if self.n_bodies:
            self.body_motion = np.array(motion[:], np.float32).reshape(-1, 6)
        if self.solver == "pbd":
            self.pbd_last_dt = self._state_pdt.value if self._state_pdt.value > 0.0 else None
            self.pos_last_init = bool(self._state_pinit.value)
        self.heat_substeps = 0
        self.it_div = self.it_den = 0
        self._scene = None
        check(self.L.sphk_checkpoint_invalidate(self.ctx), "sphk_checkpoint_invalidate")
        if getattr(self, "adaptive", False):
            self.measure_speed()
        if self._tank is not None:   # the frame time of the saved run
            check(self.L.sphk_tank_set_time(self.ctx, C.c_double(self.simulated_time)), "sphk_tank_set_time")
        self.synchronize()
        return u.raw[:user_b.value]

    def owned(self, t):
        """the live slots of a per-particle tensor (the reductions run over the live count, as in the class layer)"""
        return t[: self.fluid.n]
