"""Cost of one kinematic body (the sph_headless --stir paddle) on the 2M-particle scenes of bench.py (DFSPH 4+4, PBD 4
iterations).

    python tools/body_cost.py [--solvers dfsph pbd] [--omega 2] [--steps 20] [--warmup 5] [--rounds 2]

Runs the python engine (the same C-ABI sequence as the class layer) on the bench.py scene and on the same scene with the
paddle (sph_headless --stir --emit-scene: the fluid points within one spacing of the paddle are dropped), alternated --rounds
times, and prints per-step times (CUDA events around --steps steps), then, from a separate torch.profiler run, the CUDA time
per launch of the body kernels and of the kernels of the boundary search they trigger.  One JSON line per solver, with the
card name and its power limit.  Scene files go to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import engine  # noqa: E402

CLI = os.path.join(ROOT, "cpp-fluid-particles_b200", "sph_headless")
F = np.float32


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def paddle_scene(solver, omega, tmp):
    import dataclasses
    sc = pkg.scene.benchmark_scene("2m", solver)
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["2m"]
    prefix = os.path.join(tmp, "paddle")
    subprocess.run([CLI, "--box", str(box), "--block", str(nx), str(ny), str(nz), "--origin", *[repr(float(o)) for o in origin],
                    "--stir", repr(float(omega)), "--emit-scene", prefix], check=True, stdout=subprocess.DEVNULL, timeout=300)
    st = np.fromfile(prefix + ".body_state.f32", F)
    body = {"points": np.fromfile(prefix + ".body.f32", F).reshape(-1, 3), "position": st[:3].tolist(),
            "orientation": st[3:7].tolist(), "linear_velocity": st[7:10].tolist(), "angular_velocity": st[10:13].tolist()}
    fluid = np.fromfile(prefix + ".fluid.f32", F).reshape(-1, 3)
    boundary = np.fromfile(prefix + ".boundary.f32", F).reshape(-1, 3)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(fluid), boundary=np.ascontiguousarray(boundary)), [body]


def system(solver, scene):
    if scene is None:
        return engine.SphkSystem(pkg.scene.benchmark_scene("2m", solver))
    sc, bodies = scene
    return engine.SphkSystem(sc, bodies=bodies)


def timed(s, steps, warmup):
    for _ in range(warmup):
        s.step()
    s.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s.stream)
    for _ in range(steps):
        s.step()
    b.record(s.stream)
    b.synchronize()
    return a.elapsed_time(b) / steps


def kernel_times(s):
    """CUDA time per launch of the body kernels and of the boundary search's hash, sort and cell-start kernels"""
    for _ in range(2):
        s.step()
    s.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            s.bodies_step()
        s.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        name = ev.key.split("(")[0]
        if "Memcpy" in name or "Memset" in name:
            continue
        out[name[:80]] = round(t / max(ev.count, 1), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "pbd"])
    ap.add_argument("--omega", type=float, default=2.0)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    name, limit = card()
    with tempfile.TemporaryDirectory() as tmp:
        for solver in a.solvers:
            scene = paddle_scene(solver, a.omega, tmp)
            res = {"solver": solver, "scene": "2m", "omega": a.omega, "card": name, "power_limit": limit,
                   "n_fluid": {"off": pkg.scene.benchmark_scene("2m", solver).n_fluid, "on": int(scene[0].fluid.shape[0])},
                   "n_body_particles": int(scene[1][0]["points"].shape[0]), "n_static_boundary": int(scene[0].boundary.shape[0]),
                   "ms_per_step": {"off": [], "on": []}}
            for _ in range(a.rounds):
                for tag, sc in (("off", None), ("on", scene)):
                    s = system(solver, sc)
                    res["ms_per_step"][tag].append(round(timed(s, a.steps, a.warmup), 3))
                    s.close()
            s = system(solver, scene)
            res["bodies_step_kernel_us_per_launch"] = kernel_times(s)
            s.close()
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
