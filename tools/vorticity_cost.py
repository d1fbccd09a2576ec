"""Cost of vorticity confinement on the 2M-particle scenes of bench.py (DFSPH 4+4, PBD 4 iterations).

    python tools/vorticity_cost.py [--solvers dfsph pbd] [--eps 0.2] [--steps 20] [--warmup 5] [--rounds 2] [--tile]

Runs the python engine (the same C-ABI sequence as the class layer) with eps = 0 and eps > 0, alternated --rounds times,
and prints per-step times (CUDA events around --steps steps) and the per-kernel times of the sweeps (torch.profiler, CUDA
time per launch) as one JSON line per solver, with the card name and its power limit."""
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


def run(solver, eps, steps, warmup, tile):
    s = engine.SphkSystem(pkg.scene.benchmark_scene("2m", solver))
    if tile:
        s.set_option(capi.OPT_TILE, 1)
    s.vorticity_eps = eps
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
    kernels = {}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            s.step()
        s.synchronize()
    for ev in prof.key_averages():
        name = ev.key
        if "k_sweep" not in name and "k_s_copy" not in name:
            continue
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        short = name.split("(")[0].replace("k_sweep_", "").replace("sphk::", "")
        op = name[name.find("<") + 1:name.rfind(">")] if "<" in name else name
        key = short.split("<")[0] + "<" + op[:120] + ">"
        kernels[key] = round(t / max(ev.count, 1), 2)
    s.close()
    return ms, kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "pbd"])
    ap.add_argument("--eps", type=float, default=0.2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--tile", action="store_true", help="tile lists (SPHK_OPT_TILE = 1)")
    a = ap.parse_args()
    name, limit = card()
    for solver in a.solvers:
        res = {"solver": solver, "scene": "2m", "tile": a.tile, "eps": a.eps, "card": name, "power_limit": limit,
               "ms_per_step": {"off": [], "on": []}, "kernel_us_per_launch": {}}
        for _ in range(a.rounds):
            for tag, eps in (("off", 0.0), ("on", a.eps)):
                ms, k = run(solver, eps, a.steps, a.warmup, a.tile)
                res["ms_per_step"][tag].append(round(ms, 3))
                res["kernel_us_per_launch"][tag] = k
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
