"""Cost of tank motion (DESIGN.md section 2.15) on the 2M-particle scenes of bench.py.

    python tools/tank_cost.py [--solvers dfsph wcsph pbd] [--steps 20] [--warmup 3] [--rounds 2] [--scene 2m]

For every solver, alternated --rounds times in one process:
  * ms/step of the python engine (the class layer's C-ABI sequence, plain launches; CUDA events around --steps steps) without a
    motion (gravity kick) and with a rolling tank (roll 5 degrees at 1 Hz about the z axis through the bottom centre, plus a spin);
  * the per-kernel times of k_gravity (off), k_tank_begin and k_tank_force (roll) (torch.profiler, CUDA time per launch; first
    round);
  * the card's name, power limit and SM clock, read before and after the runs.
One JSON line per solver."""
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
from cpp_fluid_particles_b200 import engine  # noqa: E402

CASES = {
    "off": None,
    "roll": dict(axis=(0.0, 0.0, 1.0), pivot=(0.5, 0.0, 0.5), roll_amplitude=0.0873, roll_omega=6.283, spin=0.1),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"]


def run(solver, case, scene, steps, warmup, profile):
    sc = pkg.scene.benchmark_scene(scene, solver)
    s = engine.SphkSystem(sc)
    spec = CASES[case]
    if spec is not None:
        s.tank = dict(spec, pivot=(0.5 * sc.params.space[0], 0.0, 0.5 * sc.params.space[2]))
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
    clock = card()[2]
    kernels = {}
    if profile:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            s.step()
            s.synchronize()
        for ev in prof.key_averages():
            name = ev.key
            if not any(k in name for k in ("k_gravity", "k_tank_begin", "k_tank_force")):
                continue
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            kernels[name.split("(")[0][:100]] = {"us_per_launch": round(t / max(ev.count, 1), 2), "launches": int(ev.count)}
    stats = {"theta_t_end": float(s.tank_state()[1][0])} if spec is not None else None
    s.close()
    return ms, kernels, clock, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solvers", nargs="+", default=["dfsph", "wcsph", "pbd"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scene", default="2m")
    a = ap.parse_args()
    name, limit, clock0, max_clock = card()
    for solver in a.solvers:
        res = {"solver": solver, "scene": a.scene, "card": name, "power_limit": limit, "sm_clock_max": max_clock,
               "ms_per_step": {}, "sm_clock_after": {}, "kernels": {}, "last_stats": {}}
        for r in range(a.rounds):
            for case in CASES:
                ms, k, clock, st = run(solver, case, a.scene, a.steps, a.warmup, r == 0)
                res["ms_per_step"].setdefault(case, []).append(round(ms, 3))
                res["sm_clock_after"].setdefault(case, []).append(clock)
                if k:
                    res["kernels"][case] = k
                if st:
                    res["last_stats"][case] = st
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
