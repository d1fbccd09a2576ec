"""Cost of the implicit viscosity solve on the 2M-particle scenes of bench.py.

    python tools/implicit_viscosity_cost.py [--solvers dfsph pbd wcsph] [--nus 0.001 0.01 0.1] [--steps 10] [--warmup 3]
                                            [--rounds 2] [--graph-steps 10]

For every solver, with nu = nu_b:
  * ms/step of the python engine (the class layer's C-ABI sequence, plain launches; CUDA events around --steps steps) with the
    solve off and at each nu, alternated --rounds times;
  * the CG iterations of every solve of the timed window;
  * the per-kernel times of the solve at the largest nu (torch.profiler, CUDA time per launch);
  * the cost of the launches that return at once: the facade's step graph (class layer) with max_iter = 50 against max_iter =
    the largest iteration count seen + 1 -- the same result, fewer enqueued no-op iterations.
One JSON line per solver, with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import capi, engine  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in out.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def run_engine(solver, nu, steps, warmup, profile):
    s = engine.SphkSystem(pkg.scene.benchmark_scene("2m", solver))
    s.implicit_nu = s.implicit_nu_boundary = nu
    for _ in range(warmup):
        s.step()
    s.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s.stream)
    for _ in range(steps):
        s.step()
    b.record(s.stream)
    b.synchronize()
    ms = a.elapsed_time(b) / steps
    iters = []
    if nu > 0:
        for _ in range(steps):
            s.step()
            iters.append(s.implicit_viscosity_stats()[0])
    kernels = {}
    if profile:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            s.step()
            s.synchronize()
        for ev in prof.key_averages():
            name = ev.key
            if "Visc" not in name and "k_visc" not in name:
                continue
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            kernels[name.split("(")[0][:100]] = {"us_per_launch": round(t / max(ev.count, 1), 2), "launches": int(ev.count)}
    s.close()
    return ms, iters, kernels


def run_graph(solver, nu, max_iter, steps, warmup):
    app = capi.SphApp(pkg.scene.benchmark_scene("2m", solver))
    app.set_implicit_viscosity(nu, nu, 1e-4, max_iter)
    for _ in range(warmup):
        app.step()
    assert app.step_graph_active()
    ms = [app.step() for _ in range(steps)]
    it = app.viscosity_stats()[0]
    app.close()
    return sum(ms) / len(ms), it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "pbd", "wcsph"])
    ap.add_argument("--nus", nargs="+", type=float, default=[0.001, 0.01, 0.1])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--graph-steps", type=int, default=10)
    a = ap.parse_args()
    name, limit = card()
    for solver in a.solvers:
        res = {"solver": solver, "scene": "2m", "card": name, "power_limit": limit, "ms_per_step": {"off": []},
               "iterations": {}, "kernels_at_largest_nu": {}}
        for r in range(a.rounds):
            ms, _, _ = run_engine(solver, 0.0, a.steps, a.warmup, False)
            res["ms_per_step"]["off"].append(round(ms, 3))
            for nu in a.nus:
                prof = r == 0 and nu == max(a.nus)
                ms, it, k = run_engine(solver, nu, a.steps, a.warmup, prof)
                res["ms_per_step"].setdefault(str(nu), []).append(round(ms, 3))
                res["iterations"].setdefault(str(nu), []).extend(it)
                if prof:
                    res["kernels_at_largest_nu"] = k
        nu = max(a.nus)
        tight = max(res["iterations"][str(nu)]) + 1
        g50, it50 = run_graph(solver, nu, 50, a.graph_steps, a.warmup)
        gt, itt = run_graph(solver, nu, tight, a.graph_steps, a.warmup)
        res["graph_ms_per_step"] = {"nu": nu, "max_iter_50": round(g50, 3), f"max_iter_{tight}": round(gt, 3),
                                    "iterations": [it50, itt]}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
