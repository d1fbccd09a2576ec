"""The default list builder (k_build_list_staged: candidate windows staged in shared memory, hits batched in registers and
written as int4) against the global-memory builder (k_build_list, SPHK_OPT_STAGED_LIST_BUILD = 0): for every particle the
same count (the true count, also past the capacity) and, entry for entry, the same list -- the same global indices in the
same order and the same self padding of the last batch.  Then every list sweep sums the same pairs in the same order."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")
    return torch


def _list(s, staged, skin):
    """(counts, entries) built by one builder.  The buffer first holds a list of another radius (skin 100 %, built by the
    other builder), so an entry the builder under test fails to write cannot pass for a right one."""
    from cpp_fluid_particles_b200 import capi
    s.set_option(capi.OPT_STAGED_LIST_BUILD, 1 - staged)
    s.set_use_list(True, 1000)
    s.neighbor_list()
    s.set_option(capi.OPT_STAGED_LIST_BUILD, staged)
    s.set_use_list(True, skin)
    cnt, ent = s.neighbor_list()
    return cnt.cpu().numpy(), ent.cpu().numpy()


def assert_builders_agree(s, skin=0, lo=0, hi=None):
    """compares the lists of particles [lo, hi); returns their counts.  Leaves the default builder selected."""
    cg, eg = _list(s, 0, skin)
    cs, es = _list(s, 1, skin)
    hi = s.fluid.n if hi is None else hi
    cg, cs = cg[lo:hi], cs[lo:hi]
    assert np.array_equal(cg, cs), f"counts differ at {np.flatnonzero(cg != cs)[:8] + lo}"
    kmax = s.list_capacity
    written = np.minimum((cg + 3) // 4 * 4, kmax)                   # the entries, the self padding of the last batch included
    valid = np.arange(kmax).reshape(kmax // 4, 1, 4) < written[None, :, None]
    eg, es = eg[:, lo:hi], es[:, lo:hi]
    bad = valid & (eg != es)
    assert not bad.any(), f"entries differ for particles {np.unique(np.nonzero(bad)[1])[:8] + lo}"
    return cg


def _system(pkg, name, solver, **kw):
    from cpp_fluid_particles_b200 import engine
    return engine.SphkSystem(pkg.scene.benchmark_scene(name, solver), step0=False, **kw)


@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
@pytest.mark.parametrize("name", ["mini", "200k"])
def test_default_builder_equals_global_builder(pkg, built, name, solver):
    _gpu()
    s = _system(pkg, name, solver)
    for _ in range(2):
        s.step()
    s.search_fluid()
    cnt = assert_builders_agree(s)
    assert cnt.max() > 20
    s.close()


def test_pbd_skin_lists_with_fast_movers(pkg, built):
    """skin lists (150 per mille) of a strongly jittered PBD block whose first projections move particles past skin/2"""
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene("config0", solver="pbd", dt=0.004, max_iter=4, jitter=0.006)
    s = engine.SphkSystem(sc, step0=False)
    worst = 0.0
    for k in range(3):
        s.step()
        d = C.c_float()                             # (read before the builds below reset it)
        s.L.sphk_get_skin_displacement(s.ctx, C.byref(d))
        worst = max(worst, d.value / sc.params.radius)
        assert_builders_agree(s, skin=150)
    assert worst > 0.075, "the scene was meant to have fast movers"
    s.search_fluid()
    assert_builders_agree(s, skin=150)
    s.close()


@pytest.mark.parametrize("kmax", [32, 36])
def test_small_capacity_overflows_alike(pkg, built, kmax):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene("config0", solver="dfsph", jitter=0.004)
    s = engine.SphkSystem(sc, step0=False, list_capacity=kmax)
    cnt = assert_builders_agree(s)
    assert (cnt > kmax).any() and (cnt < kmax).any()
    s.close()


def test_active_sub_range(pkg, built):
    """a slab context's active range: lists of [begin, begin + count) only, begin not at a tile boundary"""
    _gpu()
    s = _system(pkg, "200k", "dfsph")
    s.step()
    s.search_fluid()
    n = s.fluid.n
    b, c = 1000 + 37, n // 2 - 91
    assert s.L.sphk_set_active_range(s.ctx, C.c_int(b), C.c_int(c)) == 0
    assert_builders_agree(s, lo=b, hi=b + c)
    s.close()


@pytest.mark.parametrize("solver", ["wcsph", "dfsph", "pbd"])
def test_fluid_count_changes_with_emitters_and_sinks(pkg, built, solver):
    _gpu()
    from cpp_fluid_particles_b200 import engine
    from test_gpu_open_boundaries import _open_scene
    sc, em, sinks = _open_scene(pkg, solver)
    s = engine.SphkSystem(sc, step0=False, max_fluid=sc.fluid.shape[0] + 600, emitters=[em], sinks=sinks)
    counts = set()
    for _ in range(4):
        s.step()
        s.search_fluid()
        counts.add(s.fluid.n)
        assert_builders_agree(s)
    assert len(counts) > 1, "the fluid count was meant to change"
    s.close()


def _tile_windows(s, sc):
    """records in the 9 + 9 candidate windows of every 128-particle tile, as k_build_list_staged stages them"""
    st = s.state()
    nx, ny, nz = (int(v) for v in sc.params.cell_size)
    ncells = nx * ny * nz
    keys = np.sort(st["p2c"])
    out = []
    for t in range(0, keys.shape[0], 128):
        k = keys[t:t + 128]
        k = k[k < ncells]
        if k.size == 0:
            continue
        total = 0
        for r in range(9):
            off = ((r // 3 - 1) * ny + (r % 3 - 1)) * nz
            cl, ch = max(int(k.min()) + off - 1, 0), min(int(k.max()) + off + 1, ncells - 1)
            if cl <= ch:
                total += sum(int(cs[ch + 1] - cs[cl]) for cs in (st["cell_start"], st["cell_startB"]))
        out.append(total)
    return np.array(out)


def test_dense_tiles_and_particles_outside_the_grid(pkg, built):
    """a compressed block: tiles whose candidate windows exceed the staging capacity (SPHK_BUILD_CAP = 2047 records) take
    the global-memory path, the rest of the block stays at the lattice density and is staged in the same launch.  Some
    particles sit outside the grid."""
    torch = _gpu()
    from cpp_fluid_particles_b200 import engine
    sc = pkg.scene.make_scene("config0", solver="dfsph", jitter=0.002)
    s = engine.SphkSystem(sc, step0=False, list_capacity=256)
    pos = s.state()["pos"]
    c = pos.mean(0)
    dense = pos[:, 0] > np.quantile(pos[:, 0], 0.5)
    pos[dense] = (pos[dense] - c) * np.float32(0.5) + c
    pos[::97] += np.float32(5.0)
    s.fluid.pos.copy_(torch.from_numpy(np.ascontiguousarray(pos, np.float32)))
    s.search_fluid()
    win = _tile_windows(s, sc)
    assert (win > 2047).any() and (win <= 2047).any()
    cnt = assert_builders_agree(s)
    assert cnt.max() > 96
    s.close()
