"""One slab rank on one GPU, checked against one global context.

A multi-GPU slab rank (cpp-fluid-particles_b200/slabs.py) runs the sweeps on a sub-grid with a non-zero origin, restricted to
its owned planes, with ghost values mirrored into the packed records and strays routed between ranks.  Here a rank is built
on the same GPU from the sorted arrays of a global context G:

    local set = G's sorted fluid particles of the planes [x0 - 1, x1 + 1), in G's order, plus ~50 particles of other planes
                (they belong to neither rank and sort behind cell_start[ncells]), shuffled in among them;
    boundary  = G's sorted boundary particles of the same planes, with G's masses (as SlabSystem takes them).

The stable sort keeps G's order inside every cell, and the cell and list walks visit neighbours in the same order, so every
owned particle must come out bit-identical to the same particle of G on the cell walk and the int32 lists.  On the tile
lists a tile holds other particles than in G, so a particle's route (staged list or cell walk) can differ: there every owned
element is held to the float64 bound of tests/ref64.py.  No torch.distributed and no NCCL: one GPU, one process."""
from __future__ import annotations

import ctypes as C
import dataclasses
import types

import numpy as np
import pytest

import ref64
from sweep_driver import PATHS, _config0

pytestmark = pytest.mark.gpu

F = np.float32
SENTINEL = np.uint32(0x7FBADBAD)           # a NaN payload no kernel writes
CUTS = {"interior": (8, 14), "one_plane": (10, 11), "edge": (0, 8)}   # config0's fluid fills planes 6..18; edge: ghost -1 is off-grid
N_OUTSIDERS = 50

# Entries that deliberately run over all particles of the set, whatever the active range: the per-particle updates that
# read no neighbour (gravity, advection, PBD velocities from positions, the EOS; also the PBD position update after the
# delta-pos sweep).  The record pre-passes that do the same are RECORD_PREPASSES below.
ALL_PARTICLE_ENTRIES = ("gravity", "advect", "pbd_velocity_from_positions", "pressure")


def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")
    return torch


def _bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


def _rows_differ(a, b):
    """per row (particle): do the bits of a and b differ anywhere"""
    d = np.asarray(a) != np.asarray(b)
    return d.reshape(d.shape[0], -1).any(1) if d.shape[0] else np.zeros(0, bool)


# ---- the global context and its sorted planes -------------------------------------------------------------------------------
class Global:
    """G = engine.SphkSystem on a scene, searched with the given masses (per sorted slot: the search does not permute them)."""

    def __init__(self, sc, masses: str, path=None):
        torch = _cuda()
        from cpp_fluid_particles_b200 import capi, engine
        self.capi, self.engine = capi, engine
        path = path or PATHS["cells"]
        self.path = path
        self.sc, self.p = sc, sc.params
        G = engine.SphkSystem(sc, step0=False, use_list=path.use_list, list_capacity=path.kmax)
        self.G = G
        st0 = G.state()
        perm0 = G.permutation().cpu().numpy()
        self.key = st0["p2c"][perm0]                 # key of sorted slot s: p2c is in pre-sort order (quirk Q2)
        n = G.fluid.n
        self.n = n
        m = np.full(n, self.p.m0, F)
        if masses == "random":
            m = (m * np.random.default_rng(17).uniform(0.5, 2.0, n)).astype(F)
        G.fluid.mass.copy_(torch.from_numpy(m))
        G.search_fluid()                             # sorted input: the identity permutation, masses stay with their slots
        st = G.state()
        assert np.array_equal(st["p2c"], self.key) and np.array_equal(_bits(st["pos"]), _bits(st0["pos"]))
        self.pos, self.mass = st["pos"], st["mass"]
        self.posB, self.massB, self.csB = st["posB"], st["massB"], st["cell_startB"]
        cx, cy, cz = (int(c) for c in self.p.cell_size)
        self.cs3, self.pc, self.nc = (cx, cy, cz), cy * cz, cx * cy * cz
        self.plane = np.where(self.key < self.nc, self.key // self.pc, -1)
        planes = self.csB[np.arange(cx + 1) * self.pc]
        self.bplane = np.searchsorted(planes, np.arange(self.posB.shape[0]), side="right") - 1
        self.rcp = G.device_rcp(self.p.cell_length)
        set_path(G, path)

    def close(self):
        self.G.close()

    def local_keys(self, ids, cs, origin):
        """numpy restatement of the rank's cell hash: G's key decoded, moved by the origin, re-encoded (ncells outside)"""
        k = self.key[ids].astype(np.int64)
        cx, cy, cz = self.cs3
        g = np.stack([k // self.pc, (k // cz) % cy, k % cz], 1) - np.asarray(origin)[None, :]
        inside = (k < self.nc) & np.all((g >= 0) & (g < np.asarray(cs)[None, :]), 1)
        return np.where(inside, (g[:, 0] * cs[1] + g[:, 1]) * cs[2] + g[:, 2], cs[0] * cs[1] * cs[2]).astype(np.int32)

    def plane_of(self, x):
        """the x-plane of a position as the device hash computes it (MUFU.RCP multiply, truncation)"""
        return np.trunc((np.asarray(x, F) * F(self.rcp)).astype(F)).astype(np.int64)


def set_path(s, path):
    s.set_option(s_capi().OPT_LIST_CAPACITY, path.kmax)
    s.set_option(s_capi().OPT_STAGED_LIST_BUILD, path.staged)
    s.set_option(s_capi().OPT_TILE, path.tile)
    s.set_use_list(path.use_list, path.skin)


def s_capi():
    from cpp_fluid_particles_b200 import capi
    return capi


# ---- one rank: a SphkOps on a sub-grid with an origin -----------------------------------------------------------------------
def rank_class():
    from cpp_fluid_particles_b200 import capi, engine
    from cpp_fluid_particles_b200.capi import SphkGrid, check

    class RankOps(engine.SphkOps):
        """A context on the sub-grid `cs` at cell `origin` of the global grid, with capacity-sized arrays (SlabSystem's
        layout) and the solver buffers of DFSPH and PBD."""

        def __init__(self, G: Global, cs, origin, cap: int, cap_b: int):
            torch = _cuda()
            self.L, self.p, self.device, self.stream = G.G.L, G.p, G.G.device, G.G.stream
            self.solver = "dfsph"
            self.fluid = engine.ParticleSet(np.zeros((cap, 3), F), self.device)
            self.fluid.n = 0
            self.boundary = engine.ParticleSet(np.full((1, 3), -1.0e3, F), self.device)
            self.cap, self.cap_b = cap, cap_b
            self.ctx = C.c_void_p()
            self._scene = None
            self._alloc_solver_buffers(cap)
            f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            self.lam, self.dpos, self.pos_last = f(cap), f(cap, 3), f(cap, 3)
            self.xsph_c, self.relaxation = 0.05, 0.75
            self._G = (C.c_float * 3)(*[float(x) for x in self.p.gravity])
            self._space = (C.c_float * 3)(*[float(x) for x in self.p.space])
            self._grid_tensors(cs, origin)
            check(self.L.sphk_create(C.byref(self.ctx), C.c_int(cap), C.c_int(cap_b), C.byref(self._g),
                                     C.c_void_p(self.stream.cuda_stream)), "sphk_create")

        def _grid_tensors(self, cs, origin):
            torch = _cuda()
            self.cs3, self.origin = tuple(int(c) for c in cs), tuple(int(o) for o in origin)
            self.ncells = self.cs3[0] * self.cs3[1] * self.cs3[2]
            g = SphkGrid()
            g.cell_size[:] = list(self.cs3)
            g.cell_length = self.p.cell_length
            g.origin[:] = list(self.origin)
            self._g = g
            self.cs_fluid = torch.zeros(self.ncells + 1, dtype=torch.int32, device=self.device)
            self.cs_boundary = torch.zeros(self.ncells + 1, dtype=torch.int32, device=self.device)
            self._scene = None

        def set_grid(self, cs, origin):
            self._grid_tensors(cs, origin)
            return int(self.L.sphk_set_grid(self.ctx, C.byref(self._g)))

        def load(self, pos, vel, mass, posB=None, massB=None):
            """the local set (input order), and the boundary when given; searches neither"""
            torch = _cuda()
            n = pos.shape[0]
            assert n <= self.cap
            self.fluid.n = n
            self.fluid.pos[:n] = torch.from_numpy(np.ascontiguousarray(pos, F)).to(self.device)
            self.fluid.vel[:n] = torch.from_numpy(np.ascontiguousarray(vel, F)).to(self.device)
            self.fluid.mass[:n] = torch.from_numpy(np.ascontiguousarray(mass, F)).to(self.device)
            if posB is not None:
                if posB.shape[0] == 0:                   # as SlabSystem: one far-away massless dummy
                    posB, massB = np.full((1, 3), -1.0e3, F), np.zeros(1, F)
                assert posB.shape[0] <= self.cap_b
                self.boundary = engine.ParticleSet(posB, self.device)
                self.boundary.mass.copy_(torch.from_numpy(np.ascontiguousarray(massB, F)))
            self._scene = None

        def search_rc(self, which=0) -> int:
            p = (self.fluid if which == 0 else self.boundary).abi()
            cs = self.cs_fluid if which == 0 else self.cs_boundary
            return int(self.L.sphk_neighbor_search(self.ctx, which, C.byref(p), C.c_void_p(cs.data_ptr())))

        def set_range(self, b, c):
            check(self.L.sphk_set_active_range(self.ctx, C.c_int(int(b)), C.c_int(int(c))), "sphk_set_active_range")

        def set_range_device(self, t):
            check(self.L.sphk_set_active_range_device(self.ctx, None if t is None else C.c_void_p(t.data_ptr())),
                  "sphk_set_active_range_device")

        def push(self, what, arr, b, c):
            check(self.L.sphk_push_range(self.ctx, self._s(), C.c_int(what), None if arr is None else C.c_void_p(arr.data_ptr()),
                                         C.c_int(int(b)), C.c_int(int(c))), "sphk_push_range")

    return RankOps


@dataclasses.dataclass
class Local:
    ids_in: np.ndarray        # G slot of every local particle, input order
    keys_in: np.ndarray       # its local key (restatement)
    perm: np.ndarray          # expected stable-sort permutation
    ids: np.ndarray           # G slot of every local sorted slot
    cs: np.ndarray            # expected cell_start[ncells + 1]
    bsel: np.ndarray          # G boundary slots of the rank
    x0: int
    x1: int
    pc: int

    def plane_start(self, k):
        """first sorted slot of local plane k (0: the left ghost plane, 1..w: owned, w + 1: the right ghost plane)"""
        return int(self.cs[min(k, self.x1 - self.x0 + 2) * self.pc])

    @property
    def own(self):
        return self.plane_start(1), self.plane_start(self.x1 - self.x0 + 1)


def local_set(G: Global, x0, x1, seed=5, drop_plane=None) -> Local:
    """The local set of owned planes [x0, x1) (plus ~50 outsiders shuffled in); drop_plane: leave that global plane empty."""
    cs = (x1 - x0 + 2,) + G.cs3[1:]
    origin = (x0 - 1, 0, 0)
    mine = (G.key < G.nc) & (G.plane >= x0 - 1) & (G.plane < x1 + 1)
    if drop_plane is not None:
        mine &= G.plane != drop_plane
    rng = np.random.default_rng(seed)
    other = np.flatnonzero((G.plane >= 0) & ((G.plane < x0 - 1) | (G.plane >= x1 + 1)))
    out = np.sort(rng.choice(other, N_OUTSIDERS, replace=False))
    ids_in = np.flatnonzero(mine)
    at = np.sort(rng.integers(0, ids_in.shape[0] + 1, N_OUTSIDERS))
    ids_in = np.insert(ids_in, at, out)
    keys = G.local_keys(ids_in, cs, origin)
    perm = np.argsort(keys, kind="stable")
    ncl = cs[0] * cs[1] * cs[2]
    cstart = np.searchsorted(keys[perm], np.arange(ncl + 1), side="left").astype(np.int32)
    assert cstart[ncl] == ids_in.shape[0] - N_OUTSIDERS, "the outsiders must sort behind cell_start[ncells]"
    bsel = np.flatnonzero((G.bplane >= x0 - 1) & (G.bplane < x1 + 1))
    return Local(ids_in, keys, perm, ids_in[perm], cstart, bsel, x0, x1, G.pc)


def load_local(R, G: Global, loc: Local, vel_g, boundary=True):
    """Loads the local set (masses per sorted slot, quirk Q2) and searches it (and the boundary)."""
    R.load(G.pos[loc.ids_in], vel_g[loc.ids_in], G.mass[loc.ids], G.posB[loc.bsel] if boundary else None,
           G.massB[loc.bsel] if boundary else None)
    if boundary:
        assert R.search_rc(1) == 0
    return R.search_rc(0)


def make_rank(G: Global, x0, x1, create=None):
    """a rank context on the cut [x0, x1) (created on the cut `create`, then re-targeted by sphk_set_grid when given)"""
    RankOps = rank_class()
    c0, c1 = create or (x0, x1)
    n_max = int(((G.plane >= -1)).sum())
    R = RankOps(G, (c1 - c0 + 2,) + G.cs3[1:], (c0 - 1, 0, 0), cap=n_max + 64, cap_b=G.posB.shape[0])
    if create:
        assert R.set_grid((x1 - x0 + 2,) + G.cs3[1:], (x0 - 1, 0, 0)) == 0
    return R


def check_search(R, G: Global, loc: Local, vel_g, what):
    st = R.state()
    n = loc.ids.shape[0]
    assert np.array_equal(st["p2c"][:n], loc.keys_in), f"{what}: particle2cell differs from the restatement"
    assert np.array_equal(R.permutation().cpu().numpy(), loc.perm), f"{what}: permutation"
    assert np.array_equal(_bits(st["pos"][:n]), _bits(G.pos[loc.ids])), f"{what}: sorted positions"
    assert np.array_equal(_bits(st["vel"][:n]), _bits(vel_g[loc.ids])), f"{what}: sorted velocities"
    assert np.array_equal(st["cell_start"], loc.cs), f"{what}: cell_start"


def _vel(G: Global):
    rng = np.random.default_rng(7)
    return (0.5 * np.sin(7.0 * G.pos) + 0.05 * rng.standard_normal(G.pos.shape)).astype(F)


# ==== A. sub-grid search and sphk_set_grid ===================================================================================
@pytest.mark.parametrize("masses", ["uniform", "random"])
def test_subgrid_search_and_set_grid(pkg, built, masses):
    G = Global(_config0(pkg), masses)
    try:
        vel = _vel(G)
        for name, (x0, x1) in CUTS.items():
            R = make_rank(G, x0, x1)
            try:
                loc = local_set(G, x0, x1)
                assert load_local(R, G, loc, vel) == 0
                check_search(R, G, loc, vel, f"{name} {x0}..{x1}")
                for d in (1, -1):                              # the cuts re-balance by one plane: same context
                    a, b = x0 + d, x1 + d
                    if a < 0:
                        continue
                    assert R.set_grid((b - a + 2,) + G.cs3[1:], (a - 1, 0, 0)) == 0
                    loc2 = local_set(G, a, b, seed=6)
                    assert load_local(R, G, loc2, vel) == 0
                    check_search(R, G, loc2, vel, f"{name} moved by {d:+d}")
            finally:
                R.close()
    finally:
        G.close()


def test_set_grid_widens_sort_key(pkg, built):
    """sphk_set_grid onto a grid whose keys need more radix passes than the creation grid's (more than 2^8 / 2^16 cells),
    at a particle count on CUB's multi-tile path.  The sort scratch is sized at creation: it must cover the wider key."""
    sc = pkg.scene.make_scene("200k", solver="dfsph")
    G = Global(sc, "uniform")
    try:
        assert G.n == 216000
        RankOps = rank_class()
        vel = _vel(G)
        ids = np.arange(G.n)
        _, cy, cz = G.cs3
        cases = [((1, 15, 17), (20, 10, 10), (1, 16, 17), (20, 10, 10)),      # 255 -> 272 cells: 8 -> 9 key bits
                 ((26, cy, cz), (10, 0, 0), (27, cy, cz), (10, 0, 0))]         # 65 000 -> 67 500 cells: 16 -> 17 key bits
        for cs_a, org_a, cs_b, org_b in cases:
            R = RankOps(G, cs_a, org_a, cap=G.n, cap_b=1)
            try:
                for cs, org in ((cs_a, org_a), (cs_b, org_b), (cs_a, org_a)):
                    assert R.set_grid(cs, org) == 0
                    R.load(G.pos, vel, G.mass)
                    rc = R.search_rc(0)
                    assert rc == 0, f"sphk_neighbor_search after sphk_set_grid {cs_a} -> {cs}: returned {rc}"
                    keys = G.local_keys(ids, cs, org)
                    perm = np.argsort(keys, kind="stable")
                    ncl = cs[0] * cs[1] * cs[2]
                    loc = Local(ids, keys, perm, ids[perm], np.searchsorted(keys[perm], np.arange(ncl + 1)).astype(np.int32),
                                np.zeros(0, np.int64), 0, 0, 1)
                    check_search(R, G, loc, vel, f"grid {cs} at {org}")
                    assert loc.cs[ncl] > 1000, "want a populated sub-grid"
            finally:
                R.close()
    finally:
        G.close()


# ==== B. active ranges =======================================================================================================
def _arr(s, name):
    return {"pos": s.fluid.pos, "vel": s.fluid.vel, "density": s.fluid.density, "pressure": s.fluid.pressure}.get(name) \
        if name in ("pos", "vel", "density", "pressure") else getattr(s, name)


@dataclasses.dataclass
class Sweep:
    name: str
    run: object               # f(s)
    outputs: tuple
    split: bool               # SphkOps._run may split it (sync given, split=True)
    pbd: bool = False


def _pbd(s, f, rho0):
    p = s.p
    s.p = dataclasses.replace(p, rho0=rho0)
    try:
        f()
    finally:
        s.p = p


def sweeps(rho0_pbd):
    return [
        Sweep("density", lambda s: s.density(), ("density",), False),
        Sweep("color_grad", lambda s: s.color_grad(), ("buffer3",), True),
        Sweep("viscosity", lambda s: s.viscosity(), ("buffer3", "vel"), False),
        Sweep("surface", lambda s: s.surface(), ("vel",), True),
        Sweep("pressure_force", lambda s: s.pressure_force(), ("vel",), False),
        Sweep("fused_density_color_grad", lambda s: s.fused_density_color_grad(False), ("density", "color_grad_buf"), True),
        Sweep("fused_dfsph_density_alpha_color_grad", lambda s: s.fused_density_color_grad(True),
              ("density", "alpha", "color_grad_buf"), False),
        Sweep("dfsph_density_alpha", lambda s: s.dfsph_density_alpha(), ("density", "alpha"), False),
        Sweep("dfsph_div_error", lambda s: s.dfsph_div_error(), ("error", "kappa"), True),
        Sweep("fused_density_alpha_div_error+cg", lambda s: s.fused_density_alpha_div_error(True),
              ("density", "alpha", "color_grad_buf", "error", "kappa"), True),
        Sweep("fused_density_alpha_div_error", lambda s: s.fused_density_alpha_div_error(False),
              ("density", "alpha", "error", "kappa"), True),
        Sweep("dfsph_div_correct", lambda s: s.dfsph_div_correct(), ("vel",), True),
        Sweep("dfsph_den_error", lambda s: s.dfsph_den_error(True), ("error", "kappa", "warm"), True),
        Sweep("dfsph_den_correct", lambda s: s.dfsph_den_correct(), ("vel",), True),
        Sweep("dfsph_den_correct_warm", lambda s: s.dfsph_den_correct(s.warm), ("vel",), True),   # the warm start, DFSPHSolver.cu:180
        Sweep("fused_viscosity_surface", lambda s: s.fused_viscosity_surface(), ("buffer3", "vel"), False),
        Sweep("pbd_density_lambda", lambda s: _pbd(s, s.pbd_density_lambda, rho0_pbd), ("density", "lam"), True, True),
        Sweep("pbd_delta_pos_apply", lambda s: _pbd(s, s.pbd_delta_pos_apply, rho0_pbd), ("dpos", "pos"), False, True),
        Sweep("pbd_xsph", lambda s: _pbd(s, s.pbd_xsph, rho0_pbd), ("vel",), False, True),
        Sweep("fused_pbd_xsph_color_grad", lambda s: _pbd(s, s.fused_pbd_xsph_color_grad, rho0_pbd), ("vel", "buffer3"), False, True),
    ]


class Scenario:
    """G on one path with per-particle inputs (G slot order), its outputs per sweep, and the float64 references."""

    def __init__(self, pkg, masses, path):
        torch = _cuda()
        self.torch = torch
        self.g = Global(_config0(pkg), masses, PATHS[path])
        G = self.g.G
        self.path = PATHS[path]
        n = self.g.n
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=G.device)  # noqa: E731
        G.lam, G.dpos, G.pos_last = f(n), f(n, 3), f(n, 3)            # (G is a DFSPH system: the PBD buffers, as in sweep_driver)
        G.xsph_c, G.relaxation = 0.05, 0.75
        rng = np.random.default_rng(11)
        vel = _vel(self.g)
        G.dfsph_density_alpha()
        G.color_grad()
        st = G.state()
        dens, alpha, cg = st["density"], G.alpha.cpu().numpy(), G.buffer3.cpu().numpy()
        dhi = (dens * F(1.28)).astype(F)
        self.rho0_pbd = float(F(np.median(dens)))
        self.inputs = {
            "pos": self.g.pos, "vel": vel, "density": dhi,
            "pressure": np.maximum(F(0), F(10) * (dhi - F(1))).astype(F),
            "alpha": alpha, "buffer3": cg, "color_grad_buf": cg,
            "kappa": (alpha * rng.uniform(-1e-3, 1e-3, n)).astype(F),
            "lam": rng.uniform(-2e-3, 2e-3, n).astype(F), "warm": (alpha * rng.uniform(-1e-3, 1e-3, n)).astype(F),
            "error": np.zeros(n, F), "dpos": np.zeros((n, 3), F),
        }
        self.sweeps = sweeps(self.rho0_pbd)
        self.out = {}
        for sw in self.sweeps:
            self.prime(G, self.inputs)
            sw.run(G)
            G.synchronize()
            self.out[sw.name] = {o: _arr(G, o).cpu().numpy().copy() for o in sw.outputs}
        self._pairs = None
        self._refs = {}

    def prime(self, s, arrays, ids=None):
        """inputs (gathered to `ids`), then a search (packs positions and velocities, forgets mirrored scalars)"""
        t = self.torch
        for k, v in arrays.items():
            v = v if ids is None else v[ids]
            _arr(s, k)[:v.shape[0]].copy_(t.from_numpy(np.ascontiguousarray(v)))
        s.search_fluid()

    def ref(self, sw, o, outs):
        """(R64, base) of output o of sweep sw on G's scene (outs: this run's outputs, for epilogues that read them)"""
        fused_error = o in ("error", "kappa") and sw.name.startswith("fused")
        if fused_error or (sw.name, o) not in self._refs:
            r = self._ref(sw, o, outs)
            if fused_error:
                return r
            self._refs[(sw.name, o)] = r
        return self._refs[(sw.name, o)]

    def _ref(self, sw, o, outs):
        if self._pairs is None:
            g = self.g
            A = types.SimpleNamespace(posF=g.pos, massF=g.mass, csF=g.G.state()["cell_start"], posB=g.posB, massB=g.massB,
                                      csB=g.csB, g=types.SimpleNamespace(ncells=g.nc), R=g.p.radius)
            self._pairs = ref64.Pairs(A)
        P, p, I = self._pairs, self.g.p, self.inputs
        rho0, dt = p.rho0, p.dt
        vel = I["vel"]
        if o == "density":
            return ref64.density(P), None
        if o == "alpha":
            return ref64.dfsph_density_alpha(P)[1], None
        if o in ("buffer3", "color_grad_buf") and sw.name not in ("viscosity", "fused_viscosity_surface"):
            return ref64.color_grad(P, self.rho0_pbd if sw.pbd else rho0, p.rho_boundary), None
        if o == "buffer3":
            return ref64.viscosity_dv(P, vel, rho0, p.visc, dt), None
        if o == "lam":
            return ref64.pbd_density_lambda(P, self.rho0_pbd, 0.75)[1], None
        if o == "dpos":
            return ref64.pbd_delta_pos(P, I["lam"], self.rho0_pbd), None
        if o in ("error", "kappa", "warm"):
            if sw.name == "dfsph_den_error":
                e, k = ref64.dfsph_den_error(P, vel, I["density"], I["alpha"], dt, rho0)
            else:
                dens = outs.get("density", I["density"])
                alpha = outs.get("alpha", I["alpha"])
                e, k = ref64.dfsph_div_error(P, vel, dens, alpha, dt, rho0, ref64.TAU)
            if o == "warm":                     # warm += stiffness
                return k, I["warm"]
            return (e if o == "error" else k), None
        if o == "pos":
            return None, None
        assert o == "vel"
        if sw.name == "viscosity":
            return ref64.viscosity_dv(P, vel, rho0, p.visc, dt), vel
        if sw.name == "surface":
            return ref64.surface_dv(P, I["buffer3"], rho0, p.surface_tension, p.air_pressure, dt), vel
        if sw.name == "pressure_force":
            return ref64.pressure_force_dv(P, I["density"], I["pressure"], dt), vel
        if sw.name == "dfsph_div_correct":
            return ref64.dfsph_correct_dv(P, I["kappa"]), vel
        if sw.name == "dfsph_den_correct_warm":
            return ref64.dfsph_correct_dv(P, I["warm"], dt), vel
        if sw.name == "dfsph_den_correct":
            return ref64.dfsph_correct_dv(P, I["kappa"], dt), vel
        if sw.name == "fused_viscosity_surface":
            rv = ref64.viscosity_dv(P, vel, rho0, p.visc, dt)
            rs = ref64.surface_dv(P, I["color_grad_buf"], rho0, p.surface_tension, p.air_pressure, dt)
            return ref64.R64(rv.value + rs.value, rv.mag + rs.mag, None if rs.alt is None else rv.value + rs.alt), vel
        return ref64.pbd_xsph_dv(P, vel, 0.05, self.rho0_pbd), vel

    def close(self):
        self.g.close()


def _sentinel_fill(R, names, slots):
    t = _cuda()
    for o in names:
        a = _arr(R, o)
        fill = 0 if o == "dpos" else int(np.asarray(SENTINEL, np.uint32).view(np.int32))
        idx = t.as_tensor(slots, device=a.device, dtype=t.long)
        a.view(t.int32)[idx] = fill             # as bits: a float NaN may be canonicalised on the way


def _guarded(sw):
    """outputs whose non-computed slots must keep their bits (positions: the PBD update runs over all particles)"""
    return tuple(o for o in sw.outputs if o != "pos") + (() if "vel" in sw.outputs else ("vel",))


def run_on_rank(S: Scenario, R, loc: Local, sw: Sweep, mode: str, rng_range=None):
    """One sweep on the rank under a range set by `mode` (host | device | split); returns (outputs, computed slots)."""
    t = S.torch
    S.prime(R, S.inputs, loc.ids)
    n = loc.ids.shape[0]
    b, e = rng_range or loc.own
    guarded = _guarded(sw)
    outside = np.setdiff1d(np.arange(n), np.arange(b, e))
    _sentinel_fill(R, guarded, outside)
    dev = None
    if mode == "host":
        R.set_range(b, e - b)
        sw.run(R)
    elif mode == "device":
        dev = t.tensor([b, e - b], dtype=t.int32, device=R.device)
        R.set_range_device(dev)
        sw.run(R)
    else:
        w = loc.x1 - loc.x0
        f1, l0 = loc.plane_start(2), loc.plane_start(w)
        pieces = [(b, f1), (l0, e), (f1, l0)] if w >= 2 else [(b, e)]
        for pb, pe in pieces:
            R.set_range(pb, pe - pb)
            sw.run(R)
    R.synchronize()
    if dev is not None:
        R.set_range_device(None)
        del dev
    return {o: _arr(R, o).cpu().numpy()[:n].copy() for o in set(sw.outputs) | set(guarded)}, np.arange(b, e)


def check_rank(S: Scenario, loc: Local, sw: Sweep, outs, computed, what):
    n = loc.ids.shape[0]
    own0, own1 = loc.own
    exact = not S.path.tile
    checked = computed[(computed >= own0) & (computed < own1)]
    outside = np.setdiff1d(np.arange(n), computed)
    for o in _guarded(sw):
        bits = _bits(outs[o][outside])
        want = np.uint32(0) if o == "dpos" else SENTINEL
        bad = np.flatnonzero(_rows_differ(bits, np.full_like(bits, want)))
        assert bad.size == 0, f"{what}: {o} of {bad.size} slot(s) outside the active range changed, first slot {outside[bad[0]]}"
    for o in sw.outputs:
        x = outs[o][checked]
        g = S.out[sw.name][o][loc.ids[checked]]
        if exact:
            bad = np.flatnonzero(_rows_differ(_bits(x), _bits(g)))
            assert bad.size == 0, (f"{what}: {o} differs from the global context at {bad.size} owned slot(s), first local slot "
                                   f"{checked[bad[0]]} (global {loc.ids[checked[bad[0]]]}): {x[bad[0]]} vs {g[bad[0]]}")
        else:
            full = {k: v for k, v in S.out[sw.name].items()}
            for k, v in outs.items():      # the epilogue of the fused error reads this run's density and alpha
                if k in ("density", "alpha"):
                    full[k] = full[k].copy()
                    full[k][loc.ids[checked]] = v[checked]
            ref, base = S.ref(sw, o, full)
            if ref is None:
                continue
            sel = loc.ids[checked]
            r = ref64.R64(ref.value[sel], ref.mag[sel], None if ref.alt is None else ref.alt[sel],
                          ref.floor if np.isscalar(ref.floor) else ref.floor[sel])
            fl = 0.0
            xx = x
            if base is not None:
                fl = ref64.f32_spacing(x)
                xx = np.asarray(x, np.float64) - np.asarray(base[sel], np.float64)
            ref64.assert_per_element(xx, r, ref64.TAU, f"{what}: {o} (per element vs float64)", fl)


RANK_PATHS = ["cells", "list", "list_global", "cap32", "skin", "tile", "tile_cap36"]


@pytest.mark.parametrize("masses", ["uniform", "random"])
@pytest.mark.parametrize("path", RANK_PATHS)
def test_active_range_sweeps(pkg, built, path, masses):
    """Every sweep entry on every path, with the owned range set from the host, from device memory, and as the three
    pieces (first plane, last plane, interior) SlabSystem._run may split a sweep into."""
    S = Scenario(pkg, masses, path)
    try:
        cuts = CUTS.items() if masses == "uniform" else [("interior", CUTS["interior"])]
        for cname, (x0, x1) in cuts:
            R = make_rank(S.g, x0, x1)
            try:
                set_path(R, S.path)
                loc = local_set(S.g, x0, x1)
                assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
                if loc.own[1] == loc.own[0]:
                    continue
                for sw in S.sweeps:
                    for mode in ("host", "device") + (("split",) if sw.split else ()):
                        outs, computed = run_on_rank(S, R, loc, sw, mode)
                        check_rank(S, loc, sw, outs, computed, f"{path}/{masses}/{cname}/{sw.name}/{mode}")
            finally:
                R.close()
    finally:
        S.close()


@pytest.mark.parametrize("path", ["cells", "list", "tile"])
def test_active_range_edges(pkg, built, path):
    """count 0 (returns 0, changes no bit), one particle, a begin that is not a multiple of 128 (tile sweeps start at
    begin / 128), and a range that ends at nF (outsiders included: only its owned slots are compared)."""
    S = Scenario(pkg, "random", path)
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(S.g, x0, x1)
        try:
            set_path(R, S.path)
            loc = local_set(S.g, x0, x1)
            assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
            own0, own1 = loc.own
            n = loc.ids.shape[0]
            begin = own0 + 37 if (own0 + 37) % 128 else own0 + 38
            ranges = {"empty": (own0 + 10, own0 + 10), "single": (own0 + 5, own0 + 6), "unaligned": (begin, begin + 300),
                      "to_nF": (loc.plane_start(x1 - x0), n)}
            picked = [sw for sw in S.sweeps if sw.name in ("density", "viscosity", "dfsph_div_correct", "dfsph_den_error",
                                                           "fused_density_alpha_div_error+cg", "pbd_delta_pos_apply")]
            for rname, rr in ranges.items():
                for sw in picked:
                    for mode in ("host", "device"):
                        outs, computed = run_on_rank(S, R, loc, sw, mode, rr)
                        check_rank(S, loc, sw, outs, computed, f"{path}/{rname}/{sw.name}/{mode}")
        finally:
            R.close()
    finally:
        S.close()


def test_all_particle_entries(pkg, built):
    """The entries of ALL_PARTICLE_ENTRIES update every particle of the set under an active range: a visible decision."""
    torch = _cuda()
    S = Scenario(pkg, "uniform", "list")
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(S.g, x0, x1)
        try:
            loc = local_set(S.g, x0, x1)
            assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
            n = loc.ids.shape[0]
            out = {"gravity": "vel", "advect": "pos", "pbd_velocity_from_positions": "vel", "pressure": "pressure"}
            for name in ALL_PARTICLE_ENTRIES:
                S.prime(R, S.inputs, loc.ids)
                R.pos_last[:n] = R.fluid.pos[:n] - 1e-3
                R.fluid.pressure.fill_(-123.0)
                before = _arr(R, out[name]).cpu().numpy()[:n].copy()
                R.set_range(loc.own[0], 1)
                getattr(R, name)()
                after = _arr(R, out[name]).cpu().numpy()[:n]
                changed = _rows_differ(_bits(after), _bits(before))
                assert changed[:loc.own[0]].all() and changed[loc.own[1]:].all(), f"{name}: not every particle was updated"
        finally:
            R.close()
    finally:
        S.close()


@pytest.mark.parametrize("path", ["list", "tile", "skin"])
def test_list_reuse_and_device_range_contents(pkg, built, path):
    """A sweep over a sub-range of the range the list was built for reuses it (its launch-count delta is its own launch);
    a sweep over a wider range rebuilds it and stays exact.  A device range whose contents change between two sweeps of one
    search reads lists that cover it."""
    torch = _cuda()
    S = Scenario(pkg, "random", path)
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(S.g, x0, x1)
        try:
            set_path(R, S.path)
            loc = local_set(S.g, x0, x1)
            assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
            sw = next(s for s in S.sweeps if s.name == "density")
            own0, own1 = loc.own
            first = (own0, loc.plane_start(2))
            n = loc.ids.shape[0]
            # narrow list first, then the whole owned range: must rebuild
            S.prime(R, S.inputs, loc.ids)
            R.set_range(first[0], first[1] - first[0])
            c0 = R.launch_count(); sw.run(R); c1 = R.launch_count()
            assert c1 - c0 == 2, f"first sweep after a search: build + sweep, got {c1 - c0} launches"
            _sentinel_fill(R, ("density",), np.setdiff1d(np.arange(n), np.arange(own0, own1)))
            R.set_range(own0, own1 - own0)
            sw.run(R); c2 = R.launch_count()
            assert c2 - c1 == 2, f"a wider range must rebuild the list: {c2 - c1} launches"
            R.synchronize()
            check_rank(S, loc, sw, {"density": R.fluid.density.cpu().numpy()[:n], "vel": np.full((n, 3), SENTINEL).view(F)},
                       np.arange(own0, own1), f"{path}: wider range")
            # a sub-range of the built range: no rebuild
            R.set_range(first[0] + 3, 40)
            sw.run(R); c3 = R.launch_count()
            assert c3 - c2 == 1, f"a sub-range must reuse the list: {c3 - c2} launches"
        finally:
            R.close()
        # device range: contents changed between two sweeps of one search (a fresh context: no list of an earlier build
        # lies in its memory)
        R = make_rank(S.g, x0, x1)
        try:
            set_path(R, S.path)
            assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
            S.prime(R, S.inputs, loc.ids)
            dev = torch.tensor([first[0], first[1] - first[0]], dtype=torch.int32, device=R.device)
            R.set_range_device(dev)
            sw.run(R)
            dev.copy_(torch.tensor([own0, own1 - own0], dtype=torch.int32))
            _sentinel_fill(R, ("density",), np.setdiff1d(np.arange(n), np.arange(own0, own1)))
            sw.run(R)
            R.synchronize()
            check_rank(S, loc, sw, {"density": R.fluid.density.cpu().numpy()[:n], "vel": np.full((n, 3), SENTINEL).view(F)},
                       np.arange(own0, own1), f"{path}: device range changed after the list build")
            R.set_range_device(None)
            del dev
        finally:
            R.close()
    finally:
        S.close()


def test_set_grid_grows_cells_skin_list(pkg, built):
    """A PBD skin list after sphk_set_grid grew ncells beyond the creation grid (the skin-flag buffer is re-allocated)."""
    S = Scenario(pkg, "random", "skin")
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(S.g, x0, x1, create=CUTS["one_plane"])
        try:
            set_path(R, S.path)
            loc = local_set(S.g, x0, x1)
            assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
            for sw in S.sweeps:
                if sw.pbd:
                    outs, computed = run_on_rank(S, R, loc, sw, "host")
                    check_rank(S, loc, sw, outs, computed, f"skin after set_grid/{sw.name}")
        finally:
            R.close()
    finally:
        S.close()


# ==== C. ghost pushes ========================================================================================================
@pytest.mark.parametrize("path", ["cells", "list"])
def test_ghost_push(pkg, built, path):
    """A neighbour scalar / velocity produced by an owned sweep is stale on the ghosts until the owners' values are pushed
    (sphk_push_range); with the push the next sweep equals G's, without it the owned particles next to the ghosts differ."""
    torch = _cuda()
    S = Scenario(pkg, "random", path)
    g = S.g
    G = g.G
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(g, x0, x1)
        try:
            set_path(R, S.path)
            loc = local_set(g, x0, x1)
            assert load_local(R, g, loc, S.inputs["vel"]) == 0
            n = loc.ids.shape[0]
            own0, own1 = loc.own
            ghosts = [(loc.plane_start(0), own0), (own1, loc.plane_start(x1 - x0 + 2))]
            gidx = np.concatenate([np.arange(a, b) for a, b in ghosts])
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a))    # noqa: E731
            by = {s.name: s for s in S.sweeps}

            def pair(first, second, what, produced, pre=None):
                """G: first, then second over everything.  Rank: first (owned), G's `produced` into the ghost slices,
                push(what), second (owned).  Returns (differs-with-push, differs-without-push) of second's outputs."""
                S.prime(G, S.inputs)
                if pre: pre(G)
                by[first].run(G)
                gv = {k: _arr(G, k).cpu().numpy().copy() for k in produced}
                by[second].run(G)
                want = {o: _arr(G, o).cpu().numpy().copy() for o in by[second].outputs}
                res = []
                for do_push in (True, False):
                    S.prime(R, S.inputs, loc.ids)
                    if pre: pre(R)
                    R.set_range(own0, own1 - own0)
                    by[first].run(R)
                    for k in produced:
                        _arr(R, k)[t(gidx).long().to(R.device)] = t(gv[k][loc.ids[gidx]]).to(R.device)
                    if do_push:
                        for a, b in ghosts:
                            R.push(what, _arr(R, "kappa" if "kappa" in produced else "lam") if what & 2 else None, a, b - a)
                    by[second].run(R)
                    R.synchronize()
                    diff = 0
                    for o in by[second].outputs:
                        x = _arr(R, o).cpu().numpy()[own0:own1]
                        y = want[o][loc.ids[own0:own1]]
                        diff += int(_rows_differ(_bits(x), _bits(y)).sum())
                    res.append(diff)
                return res

            cases = [("dfsph_div_error", "dfsph_div_correct", 2, ("kappa",)),
                     ("dfsph_den_error", "dfsph_den_correct", 2, ("kappa",)),
                     ("pbd_density_lambda", "pbd_delta_pos_apply", 2, ("lam",)),
                     ("dfsph_div_correct", "viscosity", 1, ("vel",)),
                     ("dfsph_den_correct", "pbd_xsph", 1, ("vel",)),
                     ("dfsph_den_error", "dfsph_den_correct", 3, ("kappa", "vel")),
                     ("dfsph_div_correct", "fused_viscosity_surface", 3, ("kappa", "vel"))]
            if path == "cells":
                cases.append(("dfsph_den_error", "dfsph_den_correct", 7, ("kappa", "vel", "pos")))
            for first, second, what, produced in cases:
                with_push, without = pair(first, second, what, produced)
                assert with_push == 0, f"push({what}) {first} -> {second}: {with_push} owned particle(s) differ from G"
                assert without > 0, f"control {first} -> {second}: without the push the ghosts' values must matter"

            # what = 3 with both halves read: G's density stiffness AND G's velocities after the density correct go to the
            # ghosts in one push; the rank's ghost records start from garbage velocities.  The correct sweep reads the
            # scalar, the viscosity sweep after it reads the velocities: a push of either half alone leaves a difference.
            S.prime(G, S.inputs)
            by["dfsph_den_error"].run(G)
            kap = G.kappa.cpu().numpy().copy()
            by["dfsph_den_correct"].run(G)
            vel = G.fluid.vel.cpu().numpy().copy()
            by["viscosity"].run(G)
            want = {o: _arr(G, o).cpu().numpy().copy() for o in ("vel", "buffer3")}
            gi = t(gidx).long().to(R.device)
            diffs = {}
            for what in (3, 1, 2):
                S.prime(R, S.inputs, loc.ids)
                R.set_range(own0, own1 - own0)
                by["dfsph_den_error"].run(R)
                R.fluid.vel[gi] = R.fluid.vel[gi] * 3.0 + 0.5
                for a, b in ghosts:
                    R.push(1, None, a, b - a)
                R.kappa[gi] = t(kap[loc.ids[gidx]]).to(R.device)
                R.fluid.vel[gi] = t(vel[loc.ids[gidx]]).to(R.device)
                for a, b in ghosts:
                    R.push(what, R.kappa, a, b - a)
                by["dfsph_den_correct"].run(R)
                by["viscosity"].run(R)
                R.synchronize()
                diffs[what] = sum(int(_rows_differ(_bits(_arr(R, o).cpu().numpy()[own0:own1]),
                                                   _bits(want[o][loc.ids[own0:own1]])).sum()) for o in want)
            assert diffs[3] == 0, f"push(3): {diffs[3]} owned particle(s) differ from G"
            assert diffs[1] > 0 and diffs[2] > 0, f"one half of the mask alone must leave a difference: {diffs}"
        finally:
            R.close()
    finally:
        S.close()


# the pre-passes that mirror an API array into the records' neighbour scalar for EVERY particle of the set, ghosts included
# (a ghost's value arrives in its API slice; the sweep that gathers it under the owned range finds it in the record):
# pre-pass -> (a sweep it runs in, the array it mirrors)
RECORD_PREPASSES = {"k_s_copy": ("dfsph_div_correct", "kappa"), "k_s_copy (lambda)": ("pbd_delta_pos_apply", "lam"),
                    "k_s_cg2": ("surface", "buffer3"), "k_s_prho": ("pressure_force", "pressure")}


def test_record_prepasses_cover_ghosts(pkg, built):
    """Under the owned range, the ghosts' API values of the gathered array reach the owned results through the pre-pass:
    with G's values the owned outputs are G's (test_active_range_sweeps), with other ghost values they differ."""
    torch = _cuda()
    S = Scenario(pkg, "random", "list")
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(S.g, x0, x1)
        try:
            set_path(R, S.path)
            loc = local_set(S.g, x0, x1)
            assert load_local(R, S.g, loc, S.inputs["vel"]) == 0
            own0, own1 = loc.own
            gidx = np.r_[loc.plane_start(0):own0, own1:loc.plane_start(x1 - x0 + 2)]
            by = {s.name: s for s in S.sweeps}
            for prepass, (name, arr) in RECORD_PREPASSES.items():
                sw = by[name]
                for spoil in (False, True):
                    S.prime(R, S.inputs, loc.ids)
                    if spoil:
                        a = _arr(R, arr)
                        gi = torch.as_tensor(gidx, device=R.device)
                        a[gi] = a[gi] * 2.0 + 1e-3
                    R.set_range(own0, own1 - own0)
                    sw.run(R)
                    R.synchronize()
                    diff = sum(int(_rows_differ(_bits(_arr(R, o).cpu().numpy()[own0:own1]),
                                                _bits(S.out[name][o][loc.ids[own0:own1]])).sum()) for o in sw.outputs)
                    if spoil:
                        assert diff > 0, f"{prepass}: the ghosts' {arr} values do not reach the owned {name} results"
                    else:
                        assert diff == 0, f"{prepass}: {diff} owned particle(s) of {name} differ from G"
        finally:
            R.close()
    finally:
        S.close()


def test_ghost_position_push_on_skin_list(pkg, built):
    """PBD skin list (skin 0.15 R): a ghost moved by its owner by more than skin/2 and pushed with what = 4 raises
    sphk_get_skin_displacement and sends the owned particles in the cells around it to the cell walk, whose results equal
    G's cell walk bit for bit (among them particles that now reach the ghost but did not hold it in their skin list)."""
    from scipy.spatial import cKDTree
    torch = _cuda()
    S = Scenario(pkg, "random", "skin")
    g, G = S.g, S.g.G
    p = g.p
    R_ = float(p.radius)
    try:
        x0, x1 = CUTS["interior"]
        R = make_rank(g, x0, x1)
        try:
            set_path(R, S.path)
            loc = local_set(g, x0, x1)
            assert load_local(R, g, loc, S.inputs["vel"]) == 0
            own0, own1 = loc.own
            opos = g.pos[loc.ids[own0:own1]].astype(np.float64)
            tree = cKDTree(opos)
            shift = np.array([0.5 * R_, 0.0, 0.0])                  # 0.5 R > skin / 2 = 0.075 R
            gain = []
            for ghost in range(own0 - 1, loc.plane_start(0) - 1, -1):   # the left ghost plane, nearest to the owned first
                old = g.pos[loc.ids[ghost]].astype(np.float64)
                near_new = set(tree.query_ball_point(old + shift, 0.999 * R_))
                near_old = set(tree.query_ball_point(old, 1.151 * R_))
                gain = sorted(near_new - near_old)
                if gain:
                    break
            assert gain, "want owned particles that reach the moved ghost but did not hold it in their skin list"
            new = (g.pos[loc.ids[ghost]] + shift.astype(F)).astype(F)
            gslot = int(loc.ids[ghost])
            # G: the cell walk with the particle moved in place (sphk_refresh: no re-sort)
            S.prime(G, S.inputs)
            G.fluid.pos[gslot] = torch.from_numpy(new).to(G.device)
            G.refresh()
            _pbd(G, G.pbd_density_lambda, S.rho0_pbd)
            want = {"density": G.fluid.density.cpu().numpy(), "lam": G.lam.cpu().numpy()}
            # rank: skin list over the owned range, then the owner's move of the ghost arrives by push
            S.prime(R, S.inputs, loc.ids)
            R.set_range(own0, own1 - own0)
            R.build_neighbor_list()
            R.fluid.pos[ghost] = torch.from_numpy(new).to(R.device)
            R.push(4, None, ghost, 1)
            d = C.c_float()
            assert int(R.L.sphk_get_skin_displacement(R.ctx, C.byref(d))) == 0
            assert d.value >= 0.49 * R_, f"skin displacement {d.value / R_:.3f} R after a 0.5 R move of a ghost"
            _pbd(R, R.pbd_density_lambda, S.rho0_pbd)
            R.synchronize()
            # owned particles in the 27 cells around the ghost's new cell walk the cells: bit-identical to G
            cell = lambda x: np.trunc((np.asarray(x, F) * F(g.rcp)).astype(F)).astype(np.int64)   # noqa: E731
            flagged = np.flatnonzero(np.all(np.abs(cell(g.pos[loc.ids[own0:own1]]) - cell(new)[None, :]) <= 1, 1)) + own0
            assert np.isin(np.asarray(gain) + own0, flagged).all()
            for o in want:
                x = _arr(R, o).cpu().numpy()[flagged]
                y = want[o][loc.ids[flagged]]
                bad = np.flatnonzero(_rows_differ(_bits(x), _bits(y)))
                assert bad.size == 0, (f"{o}: {bad.size} owned particle(s) around the moved ghost differ from G's cell walk, "
                                       f"first local slot {flagged[bad[0]]}: {x[bad[0]]} vs {y[bad[0]]}")
        finally:
            R.close()
    finally:
        S.close()


# ==== D. strays ==============================================================================================================
def _stray_args(arrays):
    k = len(arrays)
    from cpp_fluid_particles_b200.slabs import _widths
    return C.c_int(k), (C.c_void_p * k)(*[a.data_ptr() for a in arrays]), (C.c_int * k)(*_widths(arrays))


WIDTHS = {"dfsph": (3, 3, 1), "pbd": (3, 3, 3), "four": (3, 3, 1, 2)}


@pytest.mark.parametrize("cut", ["interior", "edge"])
@pytest.mark.parametrize("arrays", list(WIDTHS))
def test_strays_collect(pkg, built, cut, arrays):
    """sphk_strays_collect against slabs.collect_strays_host: owned particles moved by 0, +-1, +-2, +-7 planes and one to
    -1e6 after the search, with an owned plane left empty; also with more strays than the block holds."""
    torch = _cuda()
    from cpp_fluid_particles_b200 import slabs
    from cpp_fluid_particles_b200.capi import check
    g = Global(_config0(pkg), "uniform")
    try:
        x0, x1 = CUTS[cut]
        R = make_rank(g, x0, x1)
        try:
            drop = x0 + 2 if cut == "interior" else None          # the edge slab's planes 0..5 are empty already
            loc = local_set(g, x0, x1, drop_plane=drop)
            assert load_local(R, g, loc, _vel(g)) == 0
            own0, own1 = loc.own
            n = loc.ids.shape[0]
            st = R.state()
            pos = st["pos"][:n].copy()
            rng = np.random.default_rng(3)
            shift = rng.choice(np.array([0, 1, -1, 2, -2, 7, -7]), own1 - own0)
            cl = F(g.p.cell_length)
            pos[own0:own1, 0] = (pos[own0:own1, 0] + shift.astype(F) * cl).astype(F)
            pos[own0 + (own1 - own0) // 2] = F(-1.0e6)
            plane_sorted = np.searchsorted(loc.cs[np.arange(x1 - x0 + 3) * g.pc], np.arange(own0, own1), side="right") - 1
            plane_now = g.plane_of(pos[own0:own1, 0]) - (x0 - 1)
            strays = np.flatnonzero(np.abs(plane_now - plane_sorted) >= 2) + own0
            assert strays.size > 20 and (np.abs(plane_now - plane_sorted) == 1).any()
            ws = WIDTHS[arrays]
            base = [pos] + [rng.standard_normal((n, w)).astype(F) if w > 1 else rng.standard_normal(n).astype(F) for w in ws[1:]]
            for cap in (strays.size + 7, max(strays.size // 3, 1)):
                dev = [torch.from_numpy(np.ascontiguousarray(a)).to(R.device) for a in base]
                host = [a.clone() for a in dev]
                nf = slabs.stray_block_floats(cap, ws)
                block = torch.full((nf,), 7.0, dtype=torch.float32, device=R.device)
                k, ptrs, widths = _stray_args(dev)
                check(R.L.sphk_strays_collect(R.ctx, C.c_void_p(R.cs_fluid.data_ptr()), C.c_int(own0), C.c_int(own1 - own0), k,
                                              ptrs, widths, C.c_void_p(block.data_ptr()), C.c_int(cap)), "sphk_strays_collect")
                R.synchronize()
                ref = slabs.collect_strays_host(host, (own0, own1), torch.as_tensor(plane_sorted), torch.as_tensor(plane_now),
                                                strays.size)
                blk = block.cpu().numpy()
                assert int(blk[:1].view(np.int32)[0]) == strays.size, "header count"
                stride = sum(ws)
                m = min(cap, strays.size)
                rows = blk[4:4 + m * stride].reshape(m, stride)
                all_rows = ref.cpu().numpy()[4:4 + strays.size * stride].reshape(strays.size, stride)
                key = lambda r: sorted(map(bytes, np.ascontiguousarray(r).view(np.uint32)))   # noqa: E731
                rb = key(rows)
                assert len(set(rb)) == m, "collected rows must be distinct"
                assert set(rb) <= set(key(all_rows)), "collected rows must be rows of strays"
                if m == strays.size:
                    assert rb == key(all_rows), "collected rows differ from the host statement (as multisets)"
                    assert np.array_equal(_bits(blk[4 + m * stride:]), _bits(np.full(nf - 4 - m * stride, 7.0, F))), \
                        "rows beyond the count were written"
                out = [a.cpu().numpy() for a in dev]
                collected_pos = {bytes(r[:3].view(np.uint32)) for r in rows}
                out_slots = [s for s in strays if bytes(np.ascontiguousarray(pos[s]).view(np.uint32)) in collected_pos]
                assert len(out_slots) == m
                expect0 = pos.copy()
                expect0[out_slots] = F(-1.0e6)
                assert np.array_equal(_bits(out[0]), _bits(expect0)), "positions: only the collected strays move out of the world"
                for a, b in zip(out[1:], base[1:]):
                    assert np.array_equal(_bits(a), _bits(b)), "the other arrays are not changed"
                if m == strays.size:
                    assert np.array_equal(_bits(out[0]), _bits(host[0].cpu().numpy())), "positions differ from the host statement"
        finally:
            R.close()
    finally:
        g.close()


@pytest.mark.parametrize("arrays", list(WIDTHS))
def test_strays_append_and_counts(pkg, built, arrays):
    """sphk_strays_append against slabs.append_strays_host for world 3 with counts {0, capacity - 1, capacity + 5};
    sphk_strays_counts returns the three headers."""
    torch = _cuda()
    from cpp_fluid_particles_b200 import slabs
    from cpp_fluid_particles_b200.capi import check
    g = Global(_config0(pkg, 0.0), "uniform")
    try:
        R = make_rank(g, *CUTS["one_plane"])
        try:
            ws = WIDTHS[arrays]
            cap, world, dst = 37, 3, 101
            counts = [0, cap - 1, cap + 5]
            nf = slabs.stray_block_floats(cap, ws)
            rng = np.random.default_rng(9)
            gathered = rng.standard_normal(world * nf).astype(F)
            for r, c in enumerate(counts):
                gathered[r * nf:r * nf + 4] = 0.0
                gathered[r * nf:r * nf + 1].view(np.int32)[0] = c
            n = dst + world * cap + 60
            base = [rng.standard_normal((n, w)).astype(F) if w > 1 else rng.standard_normal(n).astype(F) for w in ws]
            dev = [torch.from_numpy(a).to(R.device) for a in base]
            host = [a.clone() for a in dev]
            gd = torch.from_numpy(gathered).to(R.device)
            k, ptrs, widths = _stray_args(dev)
            check(R.L.sphk_strays_append(R.ctx, C.c_void_p(gd.data_ptr()), C.c_int(world), C.c_int(cap), k, ptrs, widths, C.c_int(dst)),
                  "sphk_strays_append")
            out = (C.c_int * world)()
            check(R.L.sphk_strays_counts(R.ctx, C.c_void_p(gd.data_ptr()), C.c_int(world), C.c_int(cap), k, widths, out))
            assert list(out) == counts
            assert slabs.append_strays_host(gd, world, cap, host, dst) == world * cap
            for a, h, b in zip(dev, host, base):
                a, h = a.cpu().numpy(), h.cpu().numpy()
                assert np.array_equal(_bits(a), _bits(h)), "appended slots differ from the host statement"
                assert np.array_equal(_bits(a[:dst]), _bits(b[:dst])) and np.array_equal(_bits(a[dst + world * cap:]), _bits(b[dst + world * cap:]))
            p = dev[0].cpu().numpy()[dst:dst + world * cap].reshape(world, cap, 3)
            for r, c in enumerate(counts):
                assert np.all(p[r, min(c, cap):] == F(-1.0e6)), "unused slots must lie out of the world"
                for a in dev[1:]:
                    v = a.cpu().numpy()[dst:dst + world * cap].reshape((world, cap, -1))
                    assert np.all(v[r, min(c, cap):] == 0.0), "unused slots of the other arrays must be zero"
        finally:
            R.close()
    finally:
        g.close()
