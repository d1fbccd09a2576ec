"""Cost of CFL-adaptive time stepping on the 2M-particle scenes of bench.py (DFSPH 4+4, PBD 4).

    python tools/adaptive_dt_cost.py [--solvers dfsph pbd] [--steps 20] [--warmup 3] [--rounds 2]

For every solver, through the facade (the class layer), alternated --rounds times:
  * fixed dt with the step graph, fixed dt with plain launches, and adaptive with a bound that never binds (C = 1e6, dt_max = dt,
    so every step runs at the fixed dt): ms per step from CUDA events around --steps steps;
  * the per-launch time of k_step_speed (torch.profiler, CUDA time per launch, a run of its own);
  * the host gap at the start of each adaptive step: from the end of the previous step's k_step_speed to the next kernel (the
    wait for the speed bound, the rule and the launches of the next step's first kernel).
One JSON line per solver, with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import capi  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def make(solver, kind):
    sc = pkg.scene.benchmark_scene("2m", solver)
    app = capi.SphApp(sc)
    if kind == "plain":
        app.set_option(3, 0)
    if kind == "adaptive":
        app.set_adaptive_dt(1e6, 0.0, float(sc.params.dt))
    return app


def timed(solver, kind, steps, warmup):
    app = make(solver, kind)
    for _ in range(warmup):
        app.step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        app.step()
    e1.record()
    e1.synchronize()
    state = {"graph": app.step_graph_active()}
    if kind == "adaptive":
        state.update(app.adaptive_stats())
    app.close()
    return e0.elapsed_time(e1) / steps, state


def profiled(solver, steps, warmup):
    app = make(solver, "adaptive")
    for _ in range(warmup):
        app.step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            app.step()
        torch.cuda.synchronize()
    app.close()
    kernel = "not measured"
    for ev in prof.key_averages():
        if ev.key.split("(")[0] == "k_step_speed":
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            kernel = {"us_per_launch": round(t / max(ev.count, 1), 2), "launches": int(ev.count)}
    gaps = []
    try:
        evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > 0),
                     key=lambda e: e.time_range.start)
        for i, e in enumerate(evs[:-1]):
            if e.name.startswith("k_step_speed"):
                gaps.append(round(evs[i + 1].time_range.start - e.time_range.end, 2))
    except Exception as ex:                     # the trace layout differs: report the gap as not measured
        gaps = f"not measured ({type(ex).__name__})"
    return kernel, gaps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "pbd"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    name, limit = card()
    for solver in a.solvers:
        res = {"solver": solver, "scene": "2m", "card": name, "power_limit": limit,
               "ms_per_step": {"fixed_graph": [], "fixed_plain": [], "adaptive": []}}
        for _ in range(a.rounds):
            for kind, key in (("graph", "fixed_graph"), ("plain", "fixed_plain"), ("adaptive", "adaptive")):
                ms, state = timed(solver, kind, a.steps, a.warmup)
                res["ms_per_step"][key].append(round(ms, 3))
                res[key + "_state"] = state
        res["k_step_speed"], res["gap_after_speed_us"] = profiled(solver, 5, a.warmup)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
