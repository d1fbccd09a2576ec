"""The execution-path matrix of the sweeps.  A sweep runs along one of several paths, chosen per particle or per tile from
runtime state: the cell walk, the int32 list (staged or global builder), the list with its per-particle overflow fallback,
the skin list, the tile lists (16-bit slots of windows staged in shared memory) with their fallbacks, the uniform-mass
walk and the per-pair mass load.  Every sweep entry of the C-ABI runs on every path, on scenes chosen to reach them, and
every output is compared with the CPU oracle and, per element, with the float64 reference (tests/sweep_driver.py).
Each case asserts that its path was taken."""
import numpy as np
import pytest

from sweep_driver import PATHS, make_case, run_sweeps

pytestmark = pytest.mark.gpu

SCENES = ["config0", "config0_mass", "mini_last", "walls", "squeezed", "n1", "n31", "n33", "n129"]
# masses set by sphk_refresh alone invalidate the list: that case runs on the cell walk whatever the path option says
CASES = [(scene, path) for scene in SCENES for path in PATHS] + [("mini_refresh", "list")]


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


@pytest.mark.parametrize("scene,path", CASES)
def test_sweep_paths(pkg, built, O, scene, path):
    ratios = {}
    run_sweeps(pkg, O, make_case(pkg, scene), PATHS[path], ratios)
    print({k: f"{v:.2e}" for k, v in ratios.items()})          # largest |x - ref| / mag per output (pytest -s)


def _host_windows(key, cs, csB, n, cap_f, cell_size):
    """tile_window (csrc/sphk_sweeps.cu) restated: the 9 fluid + 9 boundary windows of every tile of particles"""
    from cpp_fluid_particles_b200.capi import TILE_PARTICLES as B, TILE_WINDOWS
    assert TILE_WINDOWS == 18
    cx, cy, cz = cell_size
    nc = cx * cy * cz
    tiles = (n + B - 1) // B
    win = np.zeros((tiles, TILE_WINDOWS, 2), np.int64)
    for t in range(tiles):
        k = key[t * B:(t + 1) * B]
        k = k[k < nc]
        if k.size == 0:
            continue
        cA, cB = int(k.min()), int(k.max())
        for w in range(18):
            r = w % 9
            off = ((r // 3 - 1) * cy + (r % 3 - 1)) * cz
            lo, hi = max(cA + off - 1, 0), min(cB + off + 1, nc - 1)
            if lo > hi:
                continue
            c = csB if w >= 9 else cs
            a, b = int(c[lo]), int(c[hi + 1])
            win[t, w] = (a + (cap_f if w >= 9 else 0), b - a)
    return win


@pytest.mark.parametrize("kmax", [96, 36, 12])
def test_tile_lists_decode_to_int32_lists(pkg, built, kmax):
    """On one search: int32 lists first, then tile lists into the same buffer.  Every slot the tile sweep reads (slots
    [0, 8 ceil(cnt/8)) of a particle on its list) decodes through the windows to the int32 list entry for entry, and the
    padding up to the end of the batch is the dummy slot T -- also for capacities that are 4 (mod 8), where the last batch
    of a nearly full list lies beyond the capacity."""
    import torch
    if not torch.cuda.is_available():
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")
    from cpp_fluid_particles_b200 import capi, engine
    sc = pkg.scene.make_scene("config0", solver="dfsph", jitter=0.005)
    s = engine.SphkSystem(sc, step0=False, list_capacity=kmax)
    try:
        s.set_option(capi.OPT_TILE, 0)
        s.set_use_list(True)
        cnt32, ent32 = s.neighbor_list()
        s.set_option(capi.OPT_TILE, 1)
        cnt, slots, win = s.tile_lists()
        cnt32, ent32 = cnt32.cpu().numpy(), ent32.cpu().numpy()
        cnt, slots, win = cnt.cpu().numpy(), slots.cpu().numpy().view(np.uint16), win.cpu().numpy()
        st = s.state()
    finally:
        s.close()
    p = sc.params
    n, nc = cnt.shape[0], p.ncells
    cs, csB = st["cell_start"], st["cell_startB"]
    key = np.searchsorted(cs, np.arange(n), side="right") - 1          # sorted cell key of each slot (ncells: outside)
    wh = _host_windows(key, cs, csB, n, n, p.cell_size)
    assert np.array_equal(win, wh), "tile windows differ from the host restatement of tile_window"
    T = wh[:, :, 1].sum(1)
    pre = np.concatenate([np.zeros((T.shape[0], 1), np.int64), np.cumsum(wh[:, :, 1], 1)], 1)
    staged = (T <= capi.TILE_CAP)[np.arange(n) // capi.TILE_PARTICLES]
    fallback = ~staged | (key >= nc)
    assert (~staged).any() and staged.any()
    assert np.all(cnt[fallback] == kmax + 1), "tiles beyond the cap and out-of-grid particles must walk the cells"
    on = ~fallback
    assert np.array_equal(cnt[on], cnt32[on]), "tile list counts differ from the int32 list counts"
    listed = np.flatnonzero(on & (cnt <= kmax))
    K = 8 * ((kmax + 7) // 8)
    k = np.arange(K)
    raw = slots[(k // 8)[None, :], listed[:, None], (k % 8)[None, :]].astype(np.int64)      # (particles, K)
    c = cnt[listed][:, None]
    read = k[None, :] < 8 * ((c + 7) // 8)                             # what k_sweep_tile reads
    if kmax % 8:
        assert (c[:, 0] > K - 8).any(), "want particles whose last batch crosses the capacity"
    t = listed // capi.TILE_PARTICLES
    tail = read & (k[None, :] >= c)
    bad = tail & (raw != T[t][:, None])
    assert not bad.any(), (f"{int(bad.sum())} padding slot(s) are not the dummy slot T, first at particle "
                           f"{listed[np.argwhere(bad)[0][0]]} slot {np.argwhere(bad)[0][1]} (cnt {c[np.argwhere(bad)[0][0], 0]})")
    entry = k[None, :] < c
    w = np.zeros_like(raw)
    for j in range(capi.TILE_WINDOWS):                                 # window of each slot
        w += raw >= pre[t, j + 1][:, None]
    w = np.minimum(w, capi.TILE_WINDOWS - 1)
    rec = wh[t[:, None], w, 0] + raw - pre[t[:, None], w]
    kk = np.minimum(k, kmax - 1)
    want = ent32[(kk // 4)[None, :], listed[:, None], (kk % 4)[None, :]].astype(np.int64)
    assert np.array_equal(np.where(entry, rec, -1), np.where(entry, want, -1)), "decoded tile lists differ from the int32 lists"
