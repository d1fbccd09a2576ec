"""Multi-rank parity check of the slab driver against a single-GPU run (rank 0 compares and prints a JSON
verdict).  Launch:  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/slab_check.py
[--backend nccl|gloo] [--scene slabtest] [--solver dfsph] [--steps 3] [--same-gpu] [--vorticity EPS]
--same-gpu puts every rank on cuda:0 (gloo, host-staged halo): lets a 1-GPU box exercise the N>1 path."""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import torch.distributed as dist
import pkgload
pkg = pkgload.load()
from cpp_fluid_particles_b200 import engine, slabs

ap = argparse.ArgumentParser()
ap.add_argument("--backend", default="nccl")
ap.add_argument("--scene", default="slabtest")
ap.add_argument("--solver", default="dfsph")
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--same-gpu", action="store_true")
ap.add_argument("--jitter", type=float, default=0.0)
ap.add_argument("--rebalance", type=int, default=-1, help="re-balance the cuts every K steps (default: the driver's own setting)")
ap.add_argument("--skew", type=int, default=0, help="start with the interior cuts this many planes off balance")
ap.add_argument("--device-scene", action="store_true", help="ranks generate their columns / the boundary shell on the device (no host arrays)")
ap.add_argument("--bullets", type=int, default=0, help="this many top-layer particles start with a velocity that carries them across "
                "several cell planes per step (what a violent impact does): exercises the stray routing")
ap.add_argument("--vorticity", type=float, default=0.0, help="vorticity confinement strength from step 1 on (0: off)")
a = ap.parse_args()
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
local = 0 if a.same_gpu else int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(local)
dist.init_process_group(a.backend)
b = pkg.scene.benchmark_scene(a.scene, a.solver)
sc = pkg.scene.make_scene(a.scene, solver=a.solver, dt=b.params.dt, max_iter=b.params.max_iter,
                          den_thr=b.params.density_error_threshold, div_thr=b.params.divergence_error_threshold, jitter=a.jitter)
sc_ranks = sc
if a.device_scene:      # the ranks build the scene on the device; the single-GPU reference below keeps the host arrays
    sc_ranks = pkg.scene.make_scene(a.scene, solver=a.solver, dt=b.params.dt, max_iter=b.params.max_iter,
                                    den_thr=b.params.density_error_threshold, div_thr=b.params.divergence_error_threshold, device_init=True)
if a.rebalance >= 0:
    os.environ["SPHK_SLAB_REBALANCE"] = str(a.rebalance)
s = slabs.SlabSystem(sc_ranks, rank, world, torch.device("cuda", local), cut_skew=a.skew)
cuts0 = list(s.cuts)
s.vorticity_eps = a.vorticity


def shoot(pos, vel):
    """Gives the chosen top-layer lattice particles (found by position: the lattice survives step 0) their bullet velocity."""
    if not a.bullets:
        return 0
    if sc.lattice is not None:
        (nx, ny, nz), origin = sc.lattice
    else:
        lo, hi = sc.fluid.min(0), sc.fluid.max(0)
        origin = tuple(float(x) for x in lo)
        nx, ny, nz = (int(round(float(hi[k] - lo[k]) / 0.02)) + 1 for k in range(3))
    idx = torch.round((pos - torch.tensor(origin, device=pos.device, dtype=pos.dtype)) / 0.02).to(torch.int64)
    speed = 30.0 * 0.004 / float(sc.params.dt)             # ~3 planes per step
    hit = 0
    for b in range(a.bullets):
        ix, iz = int((b + 0.5) * nx / a.bullets), nz // 2 + (b % 3) - 1
        m = (idx[:, 0] == ix) & (idx[:, 1] == ny - 1) & (idx[:, 2] == iz)
        v = torch.tensor([speed if b % 2 == 0 else -speed, 0.7 * speed, 0.0], device=pos.device, dtype=vel.dtype)
        if a.solver == "pbd":       # PBD derives the velocity from the positions (PBDSolver.cu:56): displace the particle instead
            pos[m] += float(sc.params.dt) * v
        else:
            vel[m] = v
        hit += int(m.sum())
    return hit


if a.bullets:
    assert a.jitter == 0.0, "--bullets finds its particles on the lattice"
    s._refresh_ranges()
    o0, o1 = s._ranges["own"]
    shoot(s.fluid.pos[o0:o1], s.fluid.vel[o0:o1])
states = [slabs.gather_state(s)]
strays = 0
for _ in range(a.steps):
    s.step()
    strays += sum(s.stray_counts())
    states.append(slabs.gather_state(s))
counts = [None] * world
s._refresh_ranges()
dist.all_gather_object(counts, (s.n_gl, s.n_own, s.n_gr, s.cuts))
if rank == 0:
    ref = engine.SphkSystem(sc, device=torch.device("cuda", local))
    ref.vorticity_eps = a.vorticity
    if a.bullets:
        assert shoot(ref.fluid.pos[:ref.fluid.n], ref.fluid.vel[:ref.fluid.n]) == a.bullets
    out = {"strays_routed": strays, "world": world, "scene": a.scene, "solver": a.solver, "counts": counts, "steps": [], "cuts_initial": cuts0, "cuts_final": list(s.cuts),
           "rebalanced": s.rebalanced, "imbalance_at_last_rebalance": s.imbalance}
    ok = True
    for k, st in enumerate(states):
        r = ref.state()
        order = np.lexsort((r["pos"][:, 2], r["pos"][:, 1], r["pos"][:, 0]))
        # canonical order is by position, which differs between the runs by ~1e-7: match through a re-sort of
        # positions rounded to 1e-4 (lattice spacing is 2e-2)
        def canon(d):
            key = np.round(d["pos"].astype(np.float64) / 2e-4).astype(np.int64)
            o = np.lexsort((key[:, 2], key[:, 1], key[:, 0]))
            return {kk: vv[o] for kk, vv in d.items() if kk in ("pos", "vel", "density")}
        cs, cr = canon(st), canon(r)
        e = {}
        for f in ("pos", "density", "vel"):
            scale = max(float(np.abs(cr[f]).max()), 1e-30)
            e[f] = float(np.abs(cs[f].astype(np.float64) - cr[f].astype(np.float64)).max() / scale)
        e["n"] = int(cs["pos"].shape[0])
        ok = ok and cs["pos"].shape == cr["pos"].shape and e["pos"] <= 1e-5 and e["density"] <= 1e-5 and e["vel"] <= 2e-4
        out["steps"].append(e)
        ref.step()
    out["ok"] = bool(ok)
    print("SLAB_CHECK " + json.dumps(out), flush=True)
s.close()
dist.barrier()
dist.destroy_process_group()
