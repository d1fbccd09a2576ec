"""Cost of probes and water-level gauges (DESIGN.md section 2.13) on the 2M-particle DFSPH scene of bench.py.

    python tools/probe_cost.py [--steps 20] [--warmup 3] [--rounds 3] [--scene 2m]

Alternated --rounds times in one process:
  * ms/step of the python engine (plain launches; CUDA events around --steps steps) with no probes and with 1024 probes plus 16
    gauges of 256 samples recorded every step;
  * the time of sphk_probe_lattice on 128^3 points and of the series record, against every kernel of the step -- its density
    sweep among them (torch.profiler, CUDA time per launch);
  * the time of one CSV drain of a frame (probe_series read back and formatted as sph_headless writes it; host clock);
  * the card's name, power limit and SM clock, read before and after the runs.
One JSON line; the spread is the list of the rounds."""
import argparse
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import engine  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"]


def probes_of(p, rng):
    """1024 probes spread over the box and 16 vertical gauges of 256 samples, upwards from the floor"""
    box = np.asarray(p.space, np.float64)
    pts = (rng.uniform(0.02, 0.97, (1024, 3)) * box).astype(np.float32)
    xz = rng.uniform(0.05, 0.95, (16, 2))
    gauges = [((float(x * box[0]), 0.002, float(z * box[2])), (float(x * box[0]), float(0.97 * box[1]), float(z * box[2])), 256)
              for x, z in xz]
    return pts, gauges


def timed_steps(s, steps):
    s.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s.stream)
    for _ in range(steps):
        s.step()
    b.record(s.stream)
    b.synchronize()
    return a.elapsed_time(b) / steps


def kernel_us(prof):
    """CUDA time per launch of every kernel of the profiled window (the step's sweeps and the probe kernels)"""
    out = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "DeviceType.CUDA" in str(ev.device_type):
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            out[ev.key.split("(")[0][:80]] = round(t / max(ev.count, 1), 1)
    return out


def drain_csv(series):
    """the CSV rows of sph_headless for one frame's series (formatting included)"""
    f = io.StringIO()
    rec, lev = series["records"].reshape(len(series["steps"]), -1), series["levels"]
    for k in range(len(series["steps"])):
        f.write(f"{series['steps'][k]},{series['times'][k]:.17g}," + ",".join(f"{x:.9g}" for x in rec[k]) + "," +
                ",".join(f"{x:.9g}" for x in lev[k]) + "\n")
    return f.getvalue()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--scene", default="2m")
    a = ap.parse_args()
    name, limit, clock0, max_clock = card()
    res = {"scene": a.scene, "solver": "dfsph", "card": name, "power_limit": limit, "sm_clock_max": max_clock, "sm_clock_before": clock0,
           "ms_per_step": {"off": [], "probes": []}, "lattice_us": [], "drain_ms": []}
    rng = np.random.default_rng(11)
    sc = pkg.scene.benchmark_scene(a.scene, "dfsph")
    pts, gauges = probes_of(sc.params, rng)
    for r in range(a.rounds):
        for case in ("off", "probes"):
            s = engine.SphkSystem(sc)
            if case == "probes":
                s.set_probes(pts, gauges, capacity=max(a.steps, 1))
            for _ in range(a.warmup):
                s.step()
            res["ms_per_step"][case].append(round(timed_steps(s, a.steps), 3))
            if case == "probes":
                t0 = time.perf_counter()
                drain_csv(s.probe_series())
                res["drain_ms"].append(round((time.perf_counter() - t0) * 1e3, 2))
                res["drain_rows"] = a.steps
                p = s.p
                sp = float(np.float32(min(p.space) / 128.0))
                s.probe_lattice((0.0, 0.0, 0.0), sp, (128, 128, 128))      # warm
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    s.step()
                    s.probe_lattice((0.0, 0.0, 0.0), sp, (128, 128, 128))
                    s.synchronize()
                k = kernel_us(prof)
                res["kernels_last_round"] = k
                res["lattice_us"].append(next((v for n, v in k.items() if "k_probe_lattice" in n), None))
            s.close()
    res["sm_clock_after"] = card()[2]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
