"""Cost and gain of DFSPH chunk activity (DESIGN.md section 4.4) over the life of the 2M-particle dam-break of bench.py.

    python tools/dfsph_activity_cost.py [--root TREE] [--scene 2m] [--ranges 1-25,30-60,100-150] [--dump DIR]

Steps the python engine (the class layer's C-ABI sequence) of the package under --root (default: this tree; another checkout
of the project gives the comparison build) from its constructor and reports, per range of steps, the mean ms/step (CUDA events
around each step) and the share of 32-particle chunks whose stiffness is exactly -0 after the range's last step (the chunks
the correct sweeps may skip while their neighbourhood is quiet too).  Early steps: the block falls freely and every chunk is
quiet; after impact at about step 26 the active share grows until, from about step 80 on, every tile is active and the
numbers give the pure cost of the checks.  --dump DIR writes pos, vel and density after the last step (.npy) for a bitwise
comparison of two builds.  One JSON line, with the card's name and power limit.

    python tools/dfsph_activity_cost.py --profile 6-25 [--scene 2m] [--root TREE]

instead steps to the first step of the range and records the range with torch.profiler (CUDA activities, a run of its own: the
tracing host is slower, so its step times are not reported).  Default 6-25: the timed window of `bench.py --gpus 1` (5 warm-up
steps after the constructor), all of it free fall.  Reports, per kernel name (templates kept, so each operator of the list
sweeps has its own line), the launches per step, the CUDA time per step and per launch, sorted by time; on stderr as a table."""
import argparse
import json
import os
import re
import subprocess
import sys


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return ["unknown"]


def profile(s, a, b):
    """Steps 1..a-1 plainly, then a..b under torch.profiler: {steps, ms_step, kernels: [{name, per_step, us_step, us_launch}]}."""
    import torch
    from torch.profiler import ProfilerActivity
    for _ in range(a - 1):
        s.step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a, b + 1):
            s.step()
        torch.cuda.synchronize()
    n = b - a + 1
    agg = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = re.sub(r"^void ", "", e.name).split("(")[0] or e.name       # kernel name with its template arguments
        t, c = agg.get(name, (0.0, 0))
        agg[name] = (t + e.time_range.elapsed_us(), c + 1)
    rows = sorted(({"name": k, "per_step": c / n, "us_step": t / n, "us_launch": t / c} for k, (t, c) in agg.items()),
                  key=lambda r: -r["us_step"])
    total = sum(r["us_step"] for r in rows)
    sys.stderr.write(f"steps {a}-{b}: {total / 1e3:.3f} ms of kernel time per step\n")
    for r in rows:
        sys.stderr.write(f"  {r['us_step']:9.1f} us/step {r['per_step']:6.2f}x {r['us_launch']:8.1f} us  {r['name']}\n")
    return {"steps": [a, b], "kernel_ms_step": total / 1e3, "kernels": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--scene", default="2m")
    ap.add_argument("--ranges", default="1-25,30-60,100-150")
    ap.add_argument("--dump", default=None)
    ap.add_argument("--profile", default=None, metavar="A-B", help="per-kernel CUDA time over steps A..B (torch.profiler)")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np
    import torch
    import pkgload
    pkg = pkgload.load()
    from cpp_fluid_particles_b200 import engine
    assert torch.cuda.is_available(), "needs a CUDA device"
    ranges = [tuple(int(x) for x in r.split("-")) for r in args.ranges.split(",")]
    s = engine.SphkSystem(pkg.scene.benchmark_scene(args.scene, "dfsph"), device=torch.device("cuda:0"))
    out = {"root": os.path.abspath(args.root), "scene": args.scene, "card": card(), "ranges": []}
    if args.profile:
        out.pop("ranges")
        out["profile"] = profile(s, *(int(x) for x in args.profile.split("-")))
        print(json.dumps(out), flush=True)
        return
    step = 0
    for a, b in ranges:
        while step < a - 1:
            s.step(); step += 1
        evs = []
        while step < b:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); s.step(); e1.record(); evs.append((e0, e1)); step += 1
        torch.cuda.synchronize()
        ms = [x.elapsed_time(y) for x, y in evs]
        k = s.kappa[: s.n_total()].view(torch.int32).cpu().numpy()
        n32 = k.size // 32 * 32
        quiet = (k[:n32].reshape(-1, 32) == np.int32(-2**31)).all(axis=1)
        out["ranges"].append({"steps": [a, b], "ms_step_mean": float(np.mean(ms)), "ms_step_median": float(np.median(ms)),
                              "quiet_chunk_share": float(quiet.mean())})
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        st = s.state()
        for f in ("pos", "vel", "density"):
            np.save(os.path.join(args.dump, f + ".npy"), st[f])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
