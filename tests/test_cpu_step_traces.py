"""The class layer (host/sph_api.cpp) and the python engine (engine.SphkOps) issue the same C-ABI calls in the same order, with
the same halo annotations, for every solver setting -- without a device.

Both layers are driven against recorders: the python engine's library handle `L` records each sphk_* name and its sync_* hooks
record the halo kind; the class layer is linked against a stub of every sphk_* entry of include/sphk.h (generated here, so a new
entry needs no edit) and a FieldHook records its produced() kinds (tests/step_trace_driver.cpp).  One step's sequence of calls,
each followed by the halo kinds it produced (0 = any array, 1 = velocities, 2 = neighbour scalar, 4 = positions), must be equal.
"""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess

import pytest
import torch

from util import ROOT

HOST = os.path.join(ROOT, "cpp-fluid-particles_b200", "host")

# calls the two layers legitimately issue differently: options and the neighbour list (the class layer builds the list lazily
# in the first sweep), launch counters, synchronisation, record refreshes, and the implicit-viscosity workspace size (the
# class layer asks for it when the setting is made, not in the step)
NOT_COMPARED = {"sphk_set_option", "sphk_build_neighbor_list", "sphk_launch_count", "sphk_synchronize", "sphk_refresh",
                "sphk_implicit_viscosity_work_floats"}

# solver, fused, surface, vorticity, implicit viscosity, one dynamic body, DFSPH thresholds >= 0 (otherwise fixed counts)
CONFIGS = [c for c in itertools.product(("wcsph", "dfsph", "pbd"), (1, 0), (1, 0), (0, 1), (0, 1), (0, 1), (0, 1))
           if c[0] == "dfsph" or c[6] == 0]


def config_id(c) -> str:
    return ",".join(str(x) for x in c)


def stub_source(header: str) -> str:
    """a definition of every sphk_* entry of the header that records its name and returns 0 (sphk_create: the driver's)"""
    txt = re.sub(r"/\*.*?\*/", "", open(header).read(), flags=re.S)
    out = ['#include "sphk.h"', 'extern "C" void step_trace_record(const char* name);', 'extern "C" {']
    for ret, name, args in re.findall(r"^\s*(const char\s*\*|int|void|long long)\s+(sphk_\w+)\s*\(([^;]*?)\)\s*;", txt, flags=re.M | re.S):
        if name == "sphk_create":
            continue
        value = {"void": "", "const char*": ' ""'}.get(ret.replace(" *", "*"), " 0")
        out.append(f'{ret} {name}({args}) {{ step_trace_record("{name}"); return{value}; }}')
    return "\n".join(out + ["}"]) + "\n"


@pytest.fixture(scope="module")
def class_layer_traces(tmp_path_factory):
    d = tmp_path_factory.mktemp("step_traces")
    stub = d / "sphk_stub.cpp"
    stub.write_text(stub_source(os.path.join(ROOT, "include", "sphk.h")))
    exe = str(d / "step_trace_driver")
    cxx = shutil.which("g++") or "/usr/bin/g++"
    cmd = [cxx, "-std=c++17", "-O0", "-I" + os.path.join(ROOT, "include"), "-I" + HOST, "-I/usr/local/cuda/include", "-o", exe,
           os.path.join(HOST, "sph_api.cpp"), str(stub), os.path.join(ROOT, "tests", "step_trace_driver.cpp"),
           "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe] + [config_id(c) for c in CONFIGS], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    traces = {}
    for line in r.stdout.splitlines():
        if line.startswith("TRACE "):
            _, key, *calls = line.split()
            traces[key] = calls
    assert sorted(traces) == sorted(config_id(c) for c in CONFIGS), r.stdout[-3000:]
    return traces


class _Recorder:
    """stands in for the library handle: every sphk_* call records its name and returns 0"""

    def __init__(self, trace):
        self.trace = trace

    def __getattr__(self, name):
        def call(*args):
            self.trace.append(name)
            return 0
        return call


def python_trace(config) -> list:
    """the python engine's trace of one step (after the first, so that PBD's "throwing" first call is out of the way): sphk_*
    names, halo<what> for each sync_* hook and split=<flag> for each _run"""
    import pkgload
    pkg = pkgload.load()
    from cpp_fluid_particles_b200 import engine
    solver, fused, surface, vorticity, implicit, body, thresholds = config

    class Traced(engine.SphkOps):
        def sync_vel(self):
            self.trace.append("halo1")

        def sync_scalar(self, t):
            self.trace.append("halo2")

        def sync_array(self, t):
            self.trace.append("halo0")

        def sync_positions(self):
            self.trace.append("halo4")

        def _run(self, op, sync=None, tensor=None, split=True):
            self.trace.append(f"split={split}")
            super()._run(op, sync, tensor, split)

    sc = pkg.scene.benchmark_scene("mini", solver)
    p = sc.params
    if not surface:
        p.surface_tension = p.air_pressure = 0.0
    if thresholds:
        p.density_error_threshold = p.divergence_error_threshold = 1e-3
    s = Traced()
    s.trace = []
    s.L, s.ctx, s.p, s.solver, s.device = _Recorder(s.trace), None, p, solver, torch.device("cpu")
    s.fluid, s.boundary = engine.ParticleSet(sc.fluid, s.device), engine.ParticleSet(sc.boundary, s.device)
    s.cs_fluid = torch.zeros(p.ncells + 1, dtype=torch.int32)
    s.cs_boundary = torch.zeros(p.ncells + 1, dtype=torch.int32)
    s._scene, s.use_list = None, True
    s._G, s._space = (C.c_float * 3)(*p.gravity), (C.c_float * 3)(*p.space)
    s._alloc_solver_buffers(s.fluid.n)
    s.fused = bool(fused)
    s.vorticity_eps = 0.2 if vorticity else 0.0
    s.implicit_nu = 1e-3 if implicit else 0.0
    if body:
        s.n_bodies, s.bodies_dynamic = 1, True
    s._step_body()
    s.trace.clear()
    s._step_body()
    return list(s.trace)


def compared(trace) -> list:
    """the trace without NOT_COMPARED and split flags, each sphk_bodies_react after the halo kinds of the sweep it follows (the
    class layer reports a DFSPH correction's velocity halo after the sweep's reaction, the python engine before it; no system has
    both: slab ranks, the only ones with halos, refuse bodies)"""
    out, react = [], None
    for t in trace:
        if t in NOT_COMPARED or t.startswith("split="):
            continue
        if react and not t.startswith("halo"):
            out.append(react)
            react = None
        if t == "sphk_bodies_react":
            react = t
        else:
            out.append(t)
    return out + ([react] if react else [])


@pytest.mark.parametrize("config", CONFIGS, ids=[config_id(c) for c in CONFIGS])
def test_layers_issue_the_same_calls(class_layer_traces, config):
    cpp = compared(class_layer_traces[config_id(config)])
    py = compared(python_trace(config))
    assert len(cpp) > 8
    assert py == cpp
