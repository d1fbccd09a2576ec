"""Cost of open boundaries (emitters and sinks) on the 2M-particle scenes of bench.py.

    python tools/open_boundary_cost.py [--solvers dfsph pbd wcsph] [--steps 10] [--warmup 3] [--rounds 2] [--tap 2.0] [--drain 1.0]

For every solver, through the facade (the class layer):
  * ms/step (SPHSystem::step's own CUDA events) of the open system: a 32 x 32 tap at the fluid spacing, centred above the block at
    0.85 of the box height, pointing down, and a floor drain of SIDE x 0.05 L x SIDE in the (0, 0, 0) corner (sph_headless --tap
    --drain), against the same closed system with plain launches and with its step graph, alternated --rounds times;
  * the per-launch times of the sink, emit and count-check kernels (torch.profiler, CUDA time per launch, a run of its own);
  * the gap between the end of the fluid search (the count-check kernel follows it) and the first solver kernel, per step: the
    time the GPU waits for the host to read the sinks' count.
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

F = np.float32
KERNELS = ("k_open_sinks_mark", "k_open_emit", "k_open_count_check")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def open_boundaries(tap, drain):
    box, (nx, ny, nz), origin = pkg.scene._CONFIGS["2m"]
    sp = F(pkg.scene.SPACING)
    half = F(0.5) * sp
    e = {"origin": [F(origin[0]) + half * F(nx - 1), F(0.85) * F(box), F(origin[2]) + half * F(nz - 1)], "direction": [0.0, -1.0, 0.0],
         "speed": tap, "spacing": sp, "width": 32, "height": 32}
    return [e], [((0.0, 0.0, 0.0), (drain, float(F(0.05) * F(box)), drain))]


def make(solver, kind, tap, drain):
    sc = pkg.scene.benchmark_scene("2m", solver)
    if kind == "open":
        em, sk = open_boundaries(tap, drain)
        return capi.SphApp(sc, max_fluid=sc.fluid.shape[0] + 2_000_000, emitters=em, sinks=sk)
    app = capi.SphApp(sc)
    if kind == "plain":
        app.set_option(3, 0)
    return app


def timed(solver, kind, steps, warmup, tap, drain):
    app = make(solver, kind, tap, drain)
    for _ in range(warmup):
        app.step()
    ms = [app.step() for _ in range(steps)]
    extra = {}
    if kind == "open":
        st, check = app.open_boundary_stats()
        extra = dict(st, check=check, fluid_count=app.fluid_count)
    else:
        extra = {"graph": app.step_graph_active()}
    app.close()
    return float(np.median(ms)), extra


def profiled(solver, steps, warmup, tap, drain):
    app = make(solver, "open", tap, drain)
    for _ in range(warmup):
        app.step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            app.step()
        torch.cuda.synchronize()
    app.close()
    kernels = {}
    for ev in prof.key_averages():
        if ev.key.split("(")[0] in KERNELS:
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            kernels[ev.key.split("(")[0]] = {"us_per_launch": round(t / max(ev.count, 1), 2), "launches": int(ev.count)}
    gaps = []
    try:
        evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > 0),
                     key=lambda e: e.time_range.start)
        for i, e in enumerate(evs[:-1]):
            if e.name.startswith("k_open_count_check"):
                search_end = max(x.time_range.end for x in evs[max(0, i - 8):i] if x.name.startswith("k_cell_start"))
                gaps.append(round(evs[i + 1].time_range.start - search_end, 2))
    except Exception as ex:                     # the trace layout differs: report the gap as not measured
        gaps = f"not measured ({type(ex).__name__})"
    return kernels, gaps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "pbd", "wcsph"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--tap", type=float, default=2.0)
    ap.add_argument("--drain", type=float, default=1.0)
    a = ap.parse_args()
    name, limit = card()
    for solver in a.solvers:
        res = {"solver": solver, "scene": "2m", "card": name, "power_limit": limit, "tap": "32x32 @ %g" % a.tap, "drain": a.drain,
               "ms_per_step_median": {"open": [], "closed_plain": [], "closed_graph": []}}
        for _ in range(a.rounds):
            for kind, key in (("closed_graph", "closed_graph"), ("plain", "closed_plain"), ("open", "open")):
                ms, extra = timed(solver, kind, a.steps, a.warmup, a.tap, a.drain)
                res["ms_per_step_median"][key].append(round(ms, 3))
                res[key + "_state"] = extra
        res["kernels"], res["search_to_solver_gap_us"] = profiled(solver, 3, a.warmup, a.tap, a.drain)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
