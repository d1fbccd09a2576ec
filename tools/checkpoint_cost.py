"""What a checkpoint costs on the GPU (DESIGN.md section 2.14), on the 2M-particle benchmark scenes.

  pack      the pack kernel (device staging + checksums): its device time from torch.profiler (CUDA activities)
  copy+file wall time from the save's return until the file is durable (the D2H copy on the side stream, the write, fsync, rename)
  d2h       the same device-to-host copy alone (a pinned torch copy of the payload's size), for the share of the PCIe link
  bytes     file bytes per fluid particle, per solver
  steps     the 2M DFSPH step time through the class layer without checkpoints and with one every 50 steps, in alternating arms
            that each restore the state after step 10 and time the next 100 steps; and the host time of each checkpoint() call

Prints one JSON line per part (pack, steps), each measured in a process of its own; card, power limit and SM clock are read in the same run.  Needs a GPU (no fallback)."""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12        # H100 SXM data sheet, 700 W card: a bound, not a measured rate


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    return q


def main(part, steps=100, arms=3, every=50):
    import torch
    assert torch.cuda.is_available(), "checkpoint_cost needs a CUDA device"
    import pkgload
    pkg = pkgload.load()
    from cpp_fluid_particles_b200 import capi, engine
    T0 = time.perf_counter()
    out = {"card": card()}
    tmp = tempfile.mkdtemp(prefix="ckpt_cost_")
    path = os.path.join(tmp, "state.ckpt")
    # pack time, durable time and bytes per particle, per solver (python engine: the same library entries)
    per = {}
    for solver in (("wcsph", "dfsph", "pbd") if part == "pack" else ()):
        print(solver, "building", round(time.perf_counter() - T0, 1), flush=True, file=sys.stderr)
        s = engine.SphkSystem(pkg.scene.benchmark_scene("2m", solver))
        for _ in range(3):
            s.step()
        print(solver, "built", round(time.perf_counter() - T0, 1), flush=True, file=sys.stderr)
        packs, durable = [], []
        s.save_state(path)                          # the first save allocates the staging buffers
        s.wait_state()
        from torch.profiler import ProfilerActivity, profile
        for k in range(3):
            s.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                s.save_state(path)
                t0 = time.perf_counter()
                s.wait_state()
                durable.append(time.perf_counter() - t0)
                torch.cuda.synchronize()
            packs += [e.device_time_total * 1e-6 for e in prof.key_averages() if "k_state_pack" in e.key]
        size = os.path.getsize(path)
        n = s.fluid.n
        print(solver, "done", round(time.perf_counter() - T0, 1), flush=True, file=sys.stderr)
        per[solver] = {"n_fluid": n, "file_bytes": size, "bytes_per_particle": size / n, "pack_ms": 1e3 * statistics.median(packs),
                       "pack_GBps": 2 * size / statistics.median(packs) / 1e9,
                       "pack_frac_hbm": 2 * size / statistics.median(packs) / HBM_PEAK,
                       "copy_to_durable_ms": 1e3 * statistics.median(durable)}
        s.close()
        torch.cuda.synchronize()
    if part == "pack":
        out["per_solver"] = per
        print(json.dumps(out))
        return
    # the D2H copy alone, pinned, the payload's size
    nbytes = 96 * 1024 * 1024
    dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        host.copy_(dev, non_blocking=True)
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    out["d2h_ms"] = 1e3 * statistics.median(ts[1:])
    out["d2h_GBps"] = nbytes / statistics.median(ts[1:]) / 1e9
    del dev, host
    # the class layer's step loop, alternating arms: no checkpoints / one every `every` steps
    sc = pkg.scene.benchmark_scene("2m", "dfsph")
    app = capi.SphApp(sc)
    for _ in range(10):
        app.step()
    # every arm starts from the state after step 10 (restored from a checkpoint), so that all arms time the same steps: the fixed
    # 4 + 4 iteration dam-break is not meant to run far past the impact, and later steps cost far more than these
    base = os.path.join(tmp, "base.ckpt")
    app.checkpoint(base)
    app.checkpoint_wait()
    arms_ms = {"none": [], f"every_{every}": []}
    worst = {"none": [], f"every_{every}": []}
    calls = []
    for _ in range(arms):
        for arm in arms_ms:
            app.restore(base)
            per_step = []
            t0 = time.perf_counter()
            for k in range(1, steps + 1):
                t = time.perf_counter()
                app.step()
                per_step.append(time.perf_counter() - t)
                if per_step[-1] > 0.05:
                    print(f"slow step {k} of arm {arm}: {1e3 * per_step[-1]:.1f} ms", flush=True, file=sys.stderr)
                if arm != "none" and k % every == 0:
                    t = time.perf_counter()
                    app.checkpoint(path)
                    calls.append(1e3 * (time.perf_counter() - t))
            if arm != "none":
                app.checkpoint_wait()
            print(arm, "arm", round(time.perf_counter() - T0, 1), flush=True, file=sys.stderr)
            arms_ms[arm].append(1e3 * (time.perf_counter() - t0) / steps)
            worst[arm].append(1e3 * max(per_step))
    app.close()
    out["step_ms"] = arms_ms
    out["worst_step_ms"] = worst
    out["checkpoint_call_ms"] = calls
    out["steps_per_arm"] = steps
    os.remove(path)
    os.remove(base)
    os.rmdir(tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    # two processes: the profiled pack measurement must not share a process with the timed step loop
    if len(sys.argv) > 1:
        main(sys.argv[1])
    else:
        for part in ("pack", "steps"):
            subprocess.run([sys.executable, os.path.abspath(__file__), part], check=True)
