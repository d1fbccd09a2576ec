"""GPU parity tests proper: every C-ABI entry point against the CPU restatement (oracle/) on the same
seeded inputs.  Integer work (cell keys, sort permutation, cell ranges) must be bit-exact; floating point
within 1e-5 scale-relative (north_star).  All calls go through the C-ABI (ctypes -> libsphk.so)."""
import numpy as np
import pytest

from util import assert_close, bits, relerr

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def _system(pkg, name, solver="wcsph", jitter=0.0, **kw):
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene(name, solver=solver, jitter=jitter, **{k: v for k, v in kw.items() if k in ("dt", "max_iter", "den_thr", "div_thr")})
    sys_ = engine.SphkSystem(sc, step0=False, **{k: v for k, v in kw.items() if k in ("use_list", "list_capacity")})
    return sc, sys_


@pytest.mark.parametrize("name,jitter", [("mini", 0.0), ("mini", 0.003), ("config0", 0.0), ("config0", 0.002)])
def test_neighbor_search_bit_exact(pkg, built, O, name, jitter):
    _torch()
    sc, s = _system(pkg, name, jitter=jitter)
    p = sc.params
    rcp = s.device_rcp(p.cell_length)
    g = O.grid(p.cell_size, p.cell_length, hash_rcp=rcp)
    # fluid
    pos_s, vel_s, p2c, cs, perm = O.neighbor_search(sc.fluid, np.zeros_like(sc.fluid), g)
    st = s.state()
    assert np.array_equal(st["p2c"], p2c), "particle2cell (pre-sort order, Q2) must be bit-exact"
    assert np.array_equal(s.permutation().cpu().numpy(), perm), "stable-sort permutation must be identical"
    assert np.array_equal(bits(st["pos"]), bits(pos_s)), "sorted positions must be bit-identical"
    assert np.array_equal(st["cell_start"], cs), "cellStart must be bit-exact"
    assert st["cell_start"][-1] == sc.fluid.shape[0]
    # boundary (searched once, SPHSystem.cu:69) + boundary mass (SPHSystem.cu:79-112)
    posb_s, _, p2cb, csb, _ = O.neighbor_search(sc.boundary, None, g)
    assert np.array_equal(st["p2cB"], p2cb)
    assert np.array_equal(bits(st["posB"]), bits(posb_s))
    assert np.array_equal(st["cell_startB"], csb)
    mb = O.boundary_mass(posb_s, csb, g, p.rho_boundary, p.radius)
    assert_close(st["massB"], mb, what="boundary mass")
    assert np.all(st["mass"] == np.float32(p.m0))
    s.close()


def test_search_out_of_grid_and_empty_cells(pkg, built, O):
    """Q8: particles outside the grid get key ncells, sort to the end, cellStart[ncells] counts the rest."""
    torch = _torch()
    sc, s = _system(pkg, "mini")
    p = sc.params
    pos = sc.fluid.copy()
    pos[::7] += np.float32(5.0)        # far outside the 0.5 box
    pos[3::11, 1] = np.float32(-0.2)   # negative coordinate -> truncation toward zero gives cell 0 ... but x/cl<0 -> -4
    s.fluid.pos.copy_(torch.from_numpy(pos))
    s.search_fluid()
    rcp = s.device_rcp(p.cell_length)
    g = O.grid(p.cell_size, p.cell_length, hash_rcp=rcp)
    pos_s, _, p2c, cs, perm = O.neighbor_search(pos, np.zeros_like(pos), g)
    st = s.state()
    assert np.array_equal(st["p2c"], p2c)
    assert (p2c == p.ncells).sum() > 0
    assert np.array_equal(st["cell_start"], cs)
    assert np.array_equal(bits(st["pos"]), bits(pos_s))
    assert st["cell_start"][-1] == (p2c < p.ncells).sum()
    s.close()


def _scene_arrays(O, s, p, rcp):
    st = s.state()
    g = O.grid(p.cell_size, p.cell_length, hash_rcp=rcp)
    return st, O.SceneArrays(st["pos"], st["mass"], st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius)


@pytest.mark.parametrize("use_list", [True, False])
@pytest.mark.parametrize("name,jitter", [("mini", 0.004), ("config0", 0.002)])
def test_sweeps_vs_oracle(pkg, built, O, name, jitter, use_list):
    """Each sweep kernel on identical inputs: jittered dam-break block + a smooth random velocity field (the shared driver
    of tests/sweep_driver.py; the full path matrix is tests/test_gpu_paths.py)."""
    from sweep_driver import PATHS, Case, run_sweeps
    sc = pkg.scene.make_scene(name, solver="dfsph", jitter=jitter, max_iter=4, den_thr=-1.0, div_thr=-1.0)
    run_sweeps(pkg, O, Case(name, sc, lattice_like=False), PATHS["list" if use_list else "cells"])


@pytest.mark.parametrize("name,jitter", [("mini", 0.004), ("config0", 0.002)])
def test_pbd_kernels_vs_oracle(pkg, built, O, name, jitter):
    torch = _torch()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene(name, solver="pbd", jitter=jitter, max_iter=4)
    s = engine.SphkSystem(sc, step0=False)
    s.set_use_list(False)
    p = sc.params
    # compress the block a little so that rho > rho0 somewhere and lambda != 0
    pos = s.state()["pos"]
    c = pos.mean(0)
    s.fluid.pos.copy_(torch.from_numpy(((pos - c) * np.float32(0.93) + c).astype(np.float32)))
    s.search_fluid()
    rcp = s.device_rcp(p.cell_length)
    st, A = _scene_arrays(O, s, p, rcp)
    s.pbd_density_lambda()
    d_ref, l_ref = O.pbd_density_lambda(A, p.rho0, s.relaxation)
    assert (l_ref != 0).sum() > 0
    assert_close(s.state()["density"], d_ref, what="pbd density")
    assert_close(s.lam.cpu().numpy(), l_ref, what="pbd lambda")
    s.lam.copy_(torch.from_numpy(l_ref))
    s.pbd_delta_pos_apply()
    dp_ref = O.pbd_delta_pos(A, l_ref, p.rho0)
    assert_close(s.dpos.cpu().numpy(), dp_ref, what="pbd delta pos")
    newpos = (st["pos"] + dp_ref).astype(np.float32)
    newpos = np.clip(newpos, 0.0, np.float32(0.99) * np.float32(p.space[0]))
    assert_close(s.state()["pos"], newpos, tol=1e-6, what="pbd applied positions")
    # velocity from positions + XSPH (Jacobi)
    s.pos_last.copy_(torch.from_numpy(st["pos"]))
    s.pbd_velocity_from_positions()
    pos_now = s.state()["pos"]
    v_ref = ((pos_now - st["pos"]) / np.float32(p.dt)).astype(np.float32)
    assert_close(s.state()["vel"], v_ref, what="vel from positions")
    A2 = O.SceneArrays(pos_now, st["mass"], st["cell_start"], st["posB"], st["massB"], st["cell_startB"],
                       O.grid(p.cell_size, p.cell_length, hash_rcp=rcp), p.radius)
    vel_in = s.state()["vel"]
    s.pbd_xsph()
    x_ref = O.pbd_xsph(A2, vel_in, s.xsph_c, p.rho0)
    assert_close(s.state()["vel"], x_ref, what="xsph")
    s.close()


def test_permute_and_list_stats(pkg, built, O):
    torch = _torch()
    sc, s = _system(pkg, "config0", solver="dfsph", jitter=0.002)
    n = s.fluid.n
    perm = s.permutation().cpu().numpy()
    a1 = torch.arange(n, dtype=torch.float32, device=s.device)
    a3 = torch.arange(3 * n, dtype=torch.float32, device=s.device).reshape(n, 3).contiguous()
    s.permute(a1, 1); s.permute(a3, 3)
    assert np.array_equal(a1.cpu().numpy(), perm.astype(np.float32))
    assert np.array_equal(a3.cpu().numpy(), np.arange(3 * n, dtype=np.float32).reshape(n, 3)[perm])
    stats = s.list_stats()
    assert stats["overflow"] == 0 and 20 < stats["total"] / n < 60 and stats["max"] <= 96
    s.close()


@pytest.mark.parametrize("skin", [0, 150])
def test_tuned_list_builder_equals_simple_cell_walk(pkg, built, O, skin):
    """k_build_list (row culling, z trimming, batched loads, int4 stores) must produce exactly the list of the
    generic cell walk: same counts, same entries in the same order, same self padding."""
    torch = _torch()
    from cpp_fluid_particles_b200 import capi
    sc, s = _system(pkg, "config0", solver="dfsph", jitter=0.004)
    lists = []
    s.set_option(capi.OPT_TILE, 0)
    # generic cell walk; the default builder (candidate windows staged in shared memory by bulk copies); the same from global memory
    for simple, staged in ((1, 0), (0, 1), (0, 0)):
        s.set_option(capi.OPT_SIMPLE_LIST_BUILD, simple)
        s.set_option(capi.OPT_STAGED_LIST_BUILD, staged)
        s.set_use_list(True, skin)
        s.search_fluid()
        cnt, ent = s.neighbor_list()
        lists.append((cnt.cpu().numpy(), ent.cpu().numpy()))
    (c0, e0) = lists[0]
    assert c0.max() > 20
    nb = (c0.max() + 3) // 4
    k = np.arange(nb * 4).reshape(nb, 1, 4)
    valid = k < (((c0 + 3) // 4) * 4)[None, :, None]          # entries incl. the self padding of the last batch
    for c1, e1 in lists[1:]:
        assert np.array_equal(c0, c1)
        assert np.array_equal(np.where(valid, e0[:nb, :c0.shape[0]], -1), np.where(valid, e1[:nb, :c0.shape[0]], -1))
    s.close()


@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
def test_tile_lists_reproduce_global_lists(pkg, built, O, solver):
    """SPHK_OPT_TILE = 1 (neighbour windows staged in shared memory by bulk copies, 16-bit lists) against the default
    int32 lists: the same pairs in the same order through another kernel instantiation -> equal up to FMA contraction;
    tiles whose windows exceed the staging capacity and out-of-grid particles take the exact cell-walk fallback."""
    _torch()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("config0", solver)
    a, b = engine.SphkSystem(sc, step0=False), engine.SphkSystem(sc, step0=False)
    b.set_option(capi.OPT_TILE, 1)
    for k in range(4):
        a.step(); b.step()
        sa, sb = a.state(), b.state()
        assert np.array_equal(sa["p2c"], sb["p2c"])
        assert_close(sb["pos"], sa["pos"], tol=1e-6, what=f"{solver} step {k} pos")
        assert_close(sb["density"], sa["density"], tol=1e-6, what=f"{solver} step {k} density")
        assert_close(sb["vel"], sa["vel"], tol=1e-5, what=f"{solver} step {k} vel")
    a.close(); b.close()


@pytest.mark.parametrize("stride", [5, 16])
def test_patch_mapped_sweep_blocks_change_nothing(pkg, built, O, stride):
    """SPHK_OPT_PATCH (experiment): the warps of a list-sweep block take their 32-particle chunks from four runs `stride`
    chunks apart instead of four consecutive ones.  Only the thread -> particle assignment changes (a bijection, also over
    the ragged last group): every particle is computed exactly as before, bit for bit."""
    _torch()
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.benchmark_scene("config0", "dfsph")
    a, b = engine.SphkSystem(sc, step0=False), engine.SphkSystem(sc, step0=False)
    b.set_option(capi.OPT_PATCH, stride)
    for k in range(3):
        a.step(); b.step()
        sa, sb = a.state(), b.state()
        for f in ("pos", "vel", "density", "pressure"):
            assert np.array_equal(sa[f], sb[f]), (f, k)
    a.close(); b.close()


def test_pbd_skin_list_with_fast_movers(pkg, built, O):
    """PBD moves particles inside a step (Q7); its neighbour list carries a skin and stays valid for particles that moved
    less than skin/2.  A strongly jittered block makes the first projections move many particles further than that: they
    flag their cell neighbourhood and everybody there walks the cells, the rest keeps the list.  The result must be the
    pure cell-walk result (same pairs; equal up to the order of exact zeros / FMA contraction)."""
    _torch()
    import ctypes as C
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene("config0", solver="pbd", dt=0.004, max_iter=4, jitter=0.006)
    a = engine.SphkSystem(sc, step0=False)
    b = engine.SphkSystem(sc, step0=False, use_list=False)
    worst = 0.0
    for k in range(6):
        a.step(); b.step()
        d = C.c_float()
        a.L.sphk_get_skin_displacement(a.ctx, C.byref(d))
        worst = max(worst, d.value / sc.params.radius)
        sa, sb = a.state(), b.state()
        assert np.array_equal(sa["p2c"], sb["p2c"]), f"step {k}"
        # (a missed neighbour would show at 1e-2; 5e-6 covers the rounding of two kernel instantiations on this rough scene)
        assert_close(sa["pos"], sb["pos"], tol=5e-6, what=f"pbd fast movers step {k} pos")
        assert_close(sa["density"], sb["density"], tol=5e-6, what=f"pbd fast movers step {k} density")
    assert worst > 0.075, f"the scene was meant to push particles beyond skin/2 (largest displacement {worst:.3f} R)"
    a.close(); b.close()


def test_list_overflow_falls_back_exactly(pkg, built, O):
    """A list capacity far below the neighbour count must not change results (per-particle cell-walk fallback)."""
    _torch()
    sc, s = _system(pkg, "mini", solver="dfsph", jitter=0.004, list_capacity=8)
    s.set_use_list(True)
    stats = s.list_stats()
    assert stats["overflow"] > 0
    s.density()
    d_small = s.state()["density"]
    sc2, s2 = _system(pkg, "mini", solver="dfsph", jitter=0.004, use_list=False)
    s2.set_use_list(False)
    s2.density()
    # same pairs in the same order through two instantiations of the same operator: equal up to FMA contraction
    assert relerr(d_small, s2.state()["density"]) <= 1e-6, "per-particle fallback must reproduce the cell walk"
    s.close(); s2.close()


@pytest.mark.parametrize("name", ["mini", "config0", "200k", "slabtest"])
def test_device_side_scene_bit_identical(pkg, built, name):
    """SURVEY 8f-4: sphk_scene_fluid_block / sphk_scene_boundary_shell against scene.py (= main.cpp:73-116 on the host):
    same positions bit for bit, same push order; also a column sub-range (what a slab rank generates)."""
    torch = _torch()
    from cpp_fluid_particles_b200 import capi, engine
    L = capi.sphk()
    host = pkg.scene.make_scene(name)
    dev = pkg.scene.make_scene(name, device_init=True)
    assert dev.fluid is None and dev.n_fluid == host.fluid.shape[0] and dev.n_boundary == host.boundary.shape[0]
    d = torch.device("cuda:0")
    st = torch.cuda.current_stream(d)
    f = engine.device_fluid_block(L, dev.lattice, d, st)
    b = engine.device_boundary_shell(L, dev.params, d, st)
    torch.cuda.synchronize()
    assert np.array_equal(bits(f.cpu().numpy()), bits(host.fluid)), "fluid block differs from main.cpp:76-85"
    assert np.array_equal(bits(b.cpu().numpy()), bits(host.boundary)), "boundary shell differs from main.cpp:89-116"
    (nx, ny, nz), _ = dev.lattice
    jb, jc = nx // 3, nx // 2
    sub = engine.device_fluid_block(L, dev.lattice, d, st, jb, jc).cpu().numpy()
    want = host.fluid.reshape(ny, nx, nz, 3)[:, jb:jb + jc].reshape(-1, 3)
    assert np.array_equal(bits(sub), bits(np.ascontiguousarray(want)))
    # a whole system built from the device-side scene equals the one built from the host arrays
    a, c = engine.SphkSystem(pkg.scene.benchmark_scene(name, "dfsph")), engine.SphkSystem(pkg.scene.benchmark_scene(name, "dfsph", device_init=True))
    a.step(); c.step()
    sa, sc_ = a.state(), c.state()
    assert np.array_equal(bits(sa["pos"]), bits(sc_["pos"])) and np.array_equal(bits(sa["density"]), bits(sc_["density"]))
    assert np.array_equal(bits(sa["massB"]), bits(sc_["massB"]))
    a.close(); c.close()


def test_particles_advect_raw(pkg, built):
    """Particles::advect (Particles.cu:28-36) on raw arrays."""
    import ctypes as C
    torch = _torch()
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    pos = torch.rand((1000, 3), device="cuda"); vel = torch.randn((1000, 3), device="cuda")
    ref = (pos.cpu().numpy() + np.float32(0.01) * vel.cpu().numpy()).astype(np.float32)
    assert L.sphk_particles_advect(C.c_void_p(pos.data_ptr()), C.c_void_p(vel.data_ptr()), 1000, C.c_float(0.01), None) == 0
    torch.cuda.synchronize()
    assert relerr(pos.cpu().numpy(), ref) <= 1e-6


def test_export_dots_vs_oracle(pkg, built, O):
    """generate_dots_CUDA (vbo.cu:26-44): positions copied, colour ramp of the density, all three branches."""
    torch = _torch()
    sc, s = _system(pkg, "mini", solver="wcsph", jitter=0.003)
    n = s.fluid.n
    dens = np.linspace(0.5, 1.3, n).astype(np.float32)
    s.fluid.density.copy_(torch.from_numpy(dens))
    dot, col = s.export_dots()
    rd, rc = O.export_dots(s.fluid.pos.cpu().numpy(), dens)
    assert np.array_equal(bits(dot.cpu().numpy()), bits(rd))
    assert_close(col.cpu().numpy(), rc, tol=1e-6, what="dot colours")
    s.close()


def test_errors_are_reported_not_thrown(pkg, built):
    """C-ABI error behaviour: bad arguments / bad call order return codes, never crash."""
    import ctypes as C
    _torch()
    from cpp_fluid_particles_b200 import capi
    L = capi.sphk()
    ctx = C.c_void_p()
    g = capi.SphkGrid(); g.cell_size[:] = [4, 4, 4]; g.cell_length = 0.1
    assert L.sphk_create(C.byref(ctx), 0, 0, C.byref(g), None) == -1
    assert L.sphk_create(C.byref(ctx), 16, 16, C.byref(g), None) == 0
    sc = capi.SphkScene()
    assert L.sphk_density(ctx, C.byref(sc)) == -4          # no neighbour search yet
    assert L.sphk_permute(ctx, None, 1, 16) == -1
    assert L.sphk_set_option(ctx, 99, 1) == -1
    L.sphk_destroy(ctx)
