"""Scenes from triangle meshes (DESIGN.md section 2.12) over the sphk_mesh_* entries of the C-ABI.

    m = meshes.load_obj("torus.obj", scale=0.1, translate=(0.5, 0.3, 0.5))   # the class layer's reader, through the facade
    m.properties()                  # area, volume, centroid, inertia, principal moments and axes (host, double)
    m.fill(spacing, origin)         # fluid lattice points inside the mesh (GPU)
    m.sample_surface(r)             # Poisson-disk boundary points on the surface (GPU)
    m.body(r, rel)                  # a body dict for engine.SphkSystem / capi.SphApp (GPU)

Vertices always pass through sphk_mesh_transform (scale * v + translate in float), so a mesh built here has the bits the C++ class
layer (sphb200::loadObj) and the headless app give it.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import check

# m0 / spacing^3 of the reference's scenes in float, as the headless app forms it (sphb200::kSceneFluidMassPerVolume)
FLUID_MASS_PER_VOLUME = float(np.float32(76.596750762082e-6) / (np.float32(0.02) * np.float32(0.02) * np.float32(0.02)))
PROPS = 18                           # SPHK_MESH_PROPS
CLOSED = 1                           # SPHK_MESH_CLOSED
INSIDE, NEAR = 1, 2                  # SPHK_MESH_INSIDE, SPHK_MESH_NEAR


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def transform(vertices, scale: float = 1.0, translate=(0.0, 0.0, 0.0)) -> np.ndarray:
    """scale * v + translate in float32 (sphk_mesh_transform)."""
    v = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    out = np.empty_like(v)
    check(capi.sphk().sphk_mesh_transform(_p(v), C.c_int(v.shape[0]), C.c_float(scale), (C.c_float * 3)(*map(float, translate)), _p(out)),
          "sphk_mesh_transform")
    return out


class Mesh:
    """A triangle mesh: float32 vertices (n, 3) after scale * v + translate (the identity leaves them as given), int32 triangles
    (m, 3), counter-clockwise seen from outside."""

    def __init__(self, vertices, triangles, scale: float = 1.0, translate=(0.0, 0.0, 0.0)):
        identity = float(scale) == 1.0 and all(float(t) == 0.0 for t in translate)
        self.vertices = (np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3)) if identity
                         else transform(vertices, scale, translate))
        self.triangles = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
        self._dev = None
        self._stream = None

    # ---- host --------------------------------------------------------------------------------------------------------------
    def properties(self) -> dict:
        """sphk_mesh_properties: {closed, area, volume, centroid, inertia (xx, yy, zz, xy, xz, yz per unit density about the
        centroid), principal (ascending), orientation (x, y, z, w: principal axes -> world)}, float64."""
        out = np.zeros(PROPS, np.float64)
        flags = C.c_int(0)
        check(capi.sphk().sphk_mesh_properties(_p(self.vertices), C.c_int(self.vertices.shape[0]), _p(self.triangles),
                                               C.c_int(self.triangles.shape[0]), _p(out), C.byref(flags)), "sphk_mesh_properties")
        return {"closed": bool(flags.value & CLOSED), "area": out[0], "volume": out[1], "centroid": out[2:5].copy(),
                "inertia": out[5:11].copy(), "principal": out[11:14].copy(), "orientation": out[14:18].copy()}

    # ---- device ------------------------------------------------------------------------------------------------------------
    def _mesh(self):
        import torch
        stream = torch.cuda.current_stream()
        if self._dev is None or self._stream != stream.cuda_stream:
            self.close()
            h = C.c_void_p()
            check(capi.sphk().sphk_mesh_create(C.byref(h), _p(self.vertices), C.c_int(self.vertices.shape[0]), _p(self.triangles),
                                               C.c_int(self.triangles.shape[0]), C.c_void_p(stream.cuda_stream)), "sphk_mesh_create")
            self._dev, self._stream = h, stream.cuda_stream
        return self._dev

    def classify(self, pos, clearance: float = 0.0) -> np.ndarray:
        """sphk_mesh_classify of points (n, 3): int32 flags, INSIDE | NEAR (distance <= clearance).  Closed meshes only."""
        import torch
        p = torch.as_tensor(np.ascontiguousarray(np.asarray(pos, np.float32).reshape(-1, 3))).cuda()
        flags = torch.empty(p.shape[0], dtype=torch.int32, device=p.device)
        check(capi.sphk().sphk_mesh_classify(self._mesh(), C.c_void_p(p.data_ptr()), C.c_int(p.shape[0]), C.c_float(clearance),
                                             C.c_void_p(flags.data_ptr())), "sphk_mesh_classify")
        return flags.cpu().numpy()

    def _counted(self, estimate: int, call) -> np.ndarray:
        import torch
        cap = max(int(estimate), 1024)
        while True:
            out = torch.empty((cap, 3), dtype=torch.float32, device="cuda")
            n = C.c_int(0)
            call(C.c_void_p(out.data_ptr()), cap, n)
            if n.value <= cap:
                return out[:n.value].cpu().numpy()
            cap = n.value

    def fill(self, spacing: float, origin=(0.0, 0.0, 0.0), clearance: float = 0.0) -> np.ndarray:
        """sphk_mesh_fill: the lattice points origin + spacing (j, i, k) inside and farther than clearance from the surface, in
        scene.fluid_lattice's order (float32 (n, 3))."""
        est = 1.1 * self.properties()["volume"] / float(spacing) ** 3 + 64
        o = (C.c_float * 3)(*map(float, origin))
        return self._counted(est, lambda out, cap, n: check(capi.sphk().sphk_mesh_fill(
            self._mesh(), C.c_float(spacing), o, C.c_float(clearance), out, C.c_int(cap), C.byref(n)), "sphk_mesh_fill"))

    def sample_surface(self, r: float) -> np.ndarray:
        """sphk_mesh_sample_surface: a maximal Poisson-disk sampling with minimum distance r (float32 (n, 3))."""
        est = 1.3 * self.properties()["area"] / float(r) ** 2 + 64
        return self._counted(est, lambda out, cap, n: check(capi.sphk().sphk_mesh_sample_surface(
            self._mesh(), C.c_float(r), out, C.c_int(cap), C.byref(n)), "sphk_mesh_sample_surface"))

    def body(self, r: float, rel: float, fluid_mass_per_volume: float = FLUID_MASS_PER_VOLUME) -> dict:
        """The body dict engine.SphkSystem and capi.SphApp take, as sphb200::meshBody builds it: surface samples at r in the
        principal frame, position = centroid, orientation = principal axes, mass = rel * fluid_mass_per_volume * V, inertia = the
        principal moments times that density (rel = 0: kinematic), at rest.  Bit for bit the C++ result."""
        p = self.properties()
        if not p["closed"]:
            raise ValueError("Mesh.body needs a closed mesh")
        x, y, z, w = (float(q) for q in p["orientation"])
        R = [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w), 2.0 * (x * z + y * w)],
             [2.0 * (x * y + z * w), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w)],
             [2.0 * (x * z - y * w), 2.0 * (y * z + x * w), 1.0 - 2.0 * (x * x + y * y)]]
        s = self.sample_surface(r).astype(np.float64)
        c = p["centroid"]
        d = [s[:, 0] - c[0], s[:, 1] - c[1], s[:, 2] - c[2]]
        local = np.stack([R[0][k] * d[0] + R[1][k] * d[1] + R[2][k] * d[2] for k in range(3)], 1).astype(np.float32)
        rho = float(np.float32(rel)) * float(np.float32(fluid_mass_per_volume))
        return {"points": local, "position": c.astype(np.float32), "orientation": p["orientation"].astype(np.float32),
                "linear_velocity": np.zeros(3, np.float32), "angular_velocity": np.zeros(3, np.float32),
                "mass": float(np.float32(rho * p["volume"])),
                "inertia": tuple(float(np.float32(m * rho)) for m in p["principal"])}

    def close(self):
        if self._dev is not None:
            capi.sphk().sphk_mesh_destroy(self._dev)
            self._dev = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def load_obj(path: str, scale: float = 1.0, translate=(0.0, 0.0, 0.0)) -> Mesh:
    """The class layer's OBJ reader (sph_app_load_obj); ValueError naming the line of a malformed file."""
    L = capi.app_lib()
    t = (C.c_float * 3)(*map(float, translate))
    nv, nt = C.c_int(0), C.c_int(0)
    rc = L.sph_app_load_obj(str(path).encode(), C.c_float(scale), t, None, C.c_int(0), None, C.c_int(0), C.byref(nv), C.byref(nt))
    if rc == 1:
        raise ValueError(L.sph_app_load_obj_error().decode())
    v = np.zeros((nv.value, 3), np.float32)
    f = np.zeros((nt.value, 3), np.int32)
    rc = L.sph_app_load_obj(str(path).encode(), C.c_float(scale), t, _p(v), C.c_int(nv.value), _p(f), C.c_int(nt.value), C.byref(nv),
                            C.byref(nt))
    if rc != 0:
        raise ValueError(L.sph_app_load_obj_error().decode() or f"sph_app_load_obj returned {rc}")
    return Mesh(v, f)            # the facade has applied scale and translate
