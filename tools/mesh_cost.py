"""Times the mesh scene builders (DESIGN.md section 2.12) on one GPU: sphk_mesh_transform (host), sphk_mesh_create,
sphk_mesh_classify, sphk_mesh_fill and sphk_mesh_sample_surface, for an icosphere of 327,680 triangles (radius 0.3) filled at a
spacing that gives about 2M points, and sampled at the 1 m tank's boundary spacing.  Every time is a host clock around work that
ends in a device synchronise, the median of 5 runs after one warm-up.  Prints one JSON line with the card and its power limit.

    python tools/mesh_cost.py
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _timed(fn, reps=5):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, out


def main():
    import torch
    import pkgload
    import mesh_ref as R
    pkgload.load()
    from cpp_fluid_particles_b200 import capi, meshes
    assert torch.cuda.is_available(), "mesh_cost.py needs a CUDA device"
    L = capi.sphk()
    v, f = R.icosphere(7, 0.3, (0.5, 0.5, 0.5))
    m = meshes.Mesh(np.asarray(v, np.float32), f)
    nv, nt = m.vertices.shape[0], m.triangles.shape[0]
    spacing, r = 0.0038, float(np.float32(0.99) / np.float32(2 * 25 - 1))
    out = {"triangles": nt, "vertices": nv, "fill_spacing": spacing, "sample_r": r}
    out["transform_ms"], _ = _timed(lambda: meshes.transform(m.vertices, 1.5, (0.1, 0.2, 0.3)))
    stream = torch.cuda.current_stream().cuda_stream

    def create():
        h = C.c_void_p()
        capi.check(L.sphk_mesh_create(C.byref(h), m.vertices.ctypes.data_as(C.c_void_p), nv, m.triangles.ctypes.data_as(C.c_void_p), nt,
                                      C.c_void_p(stream)), "sphk_mesh_create")
        L.sphk_mesh_destroy(h)
    out["create_ms"], _ = _timed(create)
    out["fill_ms"], pts = _timed(lambda: m.fill(spacing, (0.0, 0.0, 0.0), spacing))
    out["fill_points"] = int(len(pts))
    dev = torch.as_tensor(pts).cuda()
    flags = torch.empty(len(pts), dtype=torch.int32, device="cuda")
    h = m._mesh()
    out["classify_ms"], _ = _timed(lambda: capi.check(L.sphk_mesh_classify(h, C.c_void_p(dev.data_ptr()), len(pts), C.c_float(spacing),
                                                                           C.c_void_p(flags.data_ptr())), "sphk_mesh_classify"))
    out["classify_points"] = int(len(pts))
    out["sample_ms"], s = _timed(lambda: m.sample_surface(r))
    out["samples"] = int(len(s))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    out["gpu"] = q[0] if q else torch.cuda.get_device_name()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
