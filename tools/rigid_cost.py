"""Cost of one two-way coupled body on the 2M-particle scenes of bench.py (DFSPH 4+4, PBD 4 iterations).

    python tools/rigid_cost.py [--solvers dfsph pbd] [--steps 20] [--warmup 5] [--rounds 2] [--n-edge 57]

The body is a hollow cube of n-edge particles per edge at the fluid spacing (57: 18 818 particles, about the size of the
sph_headless --stir paddle), neutrally buoyant, at the centre of the fluid block; the fluid points within one spacing of it
are dropped.  Runs the python engine (the class layer's C-ABI sequence) on the bench.py scene and on the scene with the body,
alternated --rounds times, and prints per-step times (CUDA events around --steps steps), then, from a separate
torch.profiler run of one step, the CUDA time per launch and launches per step of the reaction and integrate kernels and of
the step's longest fluid sweep.  One JSON line per solver, with the card name and its power limit."""
import argparse
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import engine  # noqa: E402

F = np.float32
SPACING = 0.02


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def body_scene(solver, n_edge):
    sc = pkg.scene.benchmark_scene("2m", solver)
    a = (np.arange(n_edge) - 0.5 * (n_edge - 1)) * SPACING
    p = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    pts = p[(np.abs(p) > a.max() - 1e-9).any(1)].astype(F)
    lo, hi = sc.fluid.min(0), sc.fluid.max(0)
    c = 0.5 * (lo + hi)
    side = n_edge * SPACING
    M = sc.params.m0 / SPACING ** 3 * side ** 3            # neutrally buoyant (DESIGN.md section 2.4)
    body = {"points": pts, "position": c.tolist(), "orientation": [0.0, 0.0, 0.0, 1.0], "linear_velocity": [0.0] * 3,
            "angular_velocity": [0.0] * 3, "mass": float(M), "inertia": [float(M * side * side / 6)] * 3}
    d = np.maximum(np.maximum(pts.min(0) + c - sc.fluid, sc.fluid - (pts.max(0) + c)), 0)
    fluid = np.ascontiguousarray(sc.fluid[(d * d).sum(1) >= SPACING * SPACING])
    return dataclasses.replace(sc, fluid=fluid), [body]


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
    for _ in range(2):
        s.step()
    s.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        s.step()
        s.synchronize()
    out, longest = {}, ("", 0.0)
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        name = ev.key.split("(")[0]
        if "k_bodies_react" in name or "k_bodies_integrate" in name:
            out[name] = {"us_per_launch": round(t / max(ev.count, 1), 2), "launches_per_step": ev.count}
        elif "k_sweep" in name and t / max(ev.count, 1) > longest[1]:
            longest = (name[:80], round(t / max(ev.count, 1), 2))
    out["longest_fluid_sweep_us_per_launch"] = {longest[0]: longest[1]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "pbd"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--n-edge", type=int, default=57)
    a = ap.parse_args()
    name, limit = card()
    for solver in a.solvers:
        scene = body_scene(solver, a.n_edge)
        res = {"solver": solver, "scene": "2m", "card": name, "power_limit": limit,
               "n_fluid": {"off": pkg.scene.benchmark_scene("2m", solver).n_fluid, "on": int(scene[0].fluid.shape[0])},
               "n_body_particles": int(scene[1][0]["points"].shape[0]), "ms_per_step": {"off": [], "on": []}}
        for _ in range(a.rounds):
            for tag, sc in (("off", None), ("on", scene)):
                s = system(solver, sc)
                res["ms_per_step"][tag].append(round(timed(s, a.steps, a.warmup), 3))
                s.close()
        s = system(solver, scene)
        res["kernels"] = kernel_times(s)
        s.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
