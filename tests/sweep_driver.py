"""Shared driver of the sweep parity tests: every sweep entry of the C-ABI (WCSPH, DFSPH, PBD and the fused entries) on
one scene and one execution path, each output compared with the CPU oracle (scale-relative, the suite's tolerances) and
with the float64 reference tests/ref64.py (per element).  The scenes are numpy-only; torch and the library are imported
when a case runs."""
from __future__ import annotations

import dataclasses

import numpy as np

import ref64
from util import TOL, assert_close, relerr

F = np.float32
TAU = ref64.TAU


# ---- execution paths ---------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Path:
    use_list: bool = True
    kmax: int = 96
    staged: int = 1        # SPHK_OPT_STAGED_LIST_BUILD
    tile: int = 0          # SPHK_OPT_TILE
    skin: int = 0          # SPHK_OPT_LIST_SKIN (1/1000 R)


PATHS = {
    "cells": Path(use_list=False),
    "list": Path(),
    "list_global": Path(staged=0),
    "cap32": Path(kmax=32),
    "cap36": Path(kmax=36),
    "tile": Path(tile=1),
    "tile_cap36": Path(tile=1, kmax=36),
    "tile_cap12": Path(tile=1, kmax=12),
    "skin": Path(skin=150),
}


# ---- scenes ------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    name: str
    sc: object                  # scene.Scene
    mass: str = "uniform"       # uniform | random (m0 U(0.5, 2)) | last (slot n-1 only) | refresh (random, set by sphk_refresh)
    lattice_like: bool = True   # a jittered block at the lattice density (capacity and tile assertions apply)
    force_scale: float = 1.0    # widens the scale-relative pressure-force comparison with the oracle: near the walls and in the
                                # squeezed block the force sums cancel ~100-fold; the per-element bound is the binding check there


def _config0(pkg, jitter=0.005):
    # jitter 0.005 spreads the neighbour counts over 12..38 (some particles at 12, 13, 32, 33, 36, 37) and puts 25 of the
    # 162 tiles beyond the tile-staging cap
    return pkg.scene.make_scene("config0", solver="dfsph", jitter=jitter, max_iter=4, den_thr=-1.0, div_thr=-1.0)


def walls_scene(pkg, seed=3):
    """A jittered block that fills the mini box: its outer planes lie exactly at 0 and 0.99 L (the values k_advect clamps
    to), so it touches all six walls and the boundary shell; plus particles beyond L (in the grid and just outside it),
    at x = -0.02 (cell 0: the hash truncates toward zero) and at x <= -cell length (outside the grid)."""
    sc = pkg.scene.make_scene("mini", solver="dfsph", max_iter=4, den_thr=-1.0, div_thr=-1.0)
    L = F(sc.params.space[0])
    hi = L * F(0.99)
    k = 25
    g = (np.arange(k, dtype=F) * (hi / F(k - 1))).astype(F)
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.default_rng(seed)
    pos = np.clip(pos + rng.uniform(-0.003, 0.003, pos.shape).astype(F), F(0), hi).astype(F)
    idx = np.stack(np.meshgrid(*(np.arange(k),) * 3, indexing="ij"), -1).reshape(-1, 3)
    pos[idx == 0] = F(0)
    pos[idx == k - 1] = hi
    cl = F(sc.params.cell_length)
    out = []
    for axis in range(3):
        for v in (L + F(0.005), F(13.2) * cl, F(-0.02), -cl, F(-1.5) * cl):
            q = np.array([0.25, 0.2, 0.3], F)
            q[axis] = v
            out.append(q)
    pos = np.concatenate([pos, np.asarray(out, F)]).astype(F)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(pos))


def squeezed_scene(pkg):
    """config0 squeezed to x0.7 about its centre: neighbour counts above 96, tiles beyond the staging caps"""
    sc = _config0(pkg, 0.002)
    c = sc.fluid.mean(0)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(((sc.fluid - c) * F(0.7) + c).astype(F)))


def small_scene(pkg, n):
    sc = _config0(pkg)
    return dataclasses.replace(sc, fluid=np.ascontiguousarray(sc.fluid[:n]))


def make_case(pkg, name) -> Case:
    if name == "config0":
        return Case(name, _config0(pkg))
    if name == "config0_mass":
        return Case(name, _config0(pkg), mass="random")
    if name == "mini_last":
        return Case(name, pkg.scene.make_scene("mini", solver="dfsph", jitter=0.004, max_iter=4, den_thr=-1.0, div_thr=-1.0),
                    mass="last", lattice_like=False)
    if name == "mini_refresh":
        return Case(name, pkg.scene.make_scene("mini", solver="dfsph", jitter=0.004, max_iter=4, den_thr=-1.0, div_thr=-1.0),
                    mass="refresh", lattice_like=False)
    if name == "walls":
        return Case(name, walls_scene(pkg), lattice_like=False, force_scale=10.0)
    if name == "squeezed":
        return Case(name, squeezed_scene(pkg), lattice_like=False, force_scale=10.0)
    if name.startswith("n"):
        return Case(name, small_scene(pkg, int(name[1:])), lattice_like=False)
    raise KeyError(name)


def case_masses(case, n, m0):
    m = np.full(n, m0, F)
    if case.mass in ("random", "refresh"):
        m = (m * np.random.default_rng(17).uniform(0.5, 2.0, n)).astype(F)
    elif case.mass == "last":
        m[n - 1] = F(4.0) * F(m0)
    return m


# ---- the driver --------------------------------------------------------------------------------------------------------------
def _check(x, oracle, ref, what, tol=TOL, floor=0.0, base=None):
    """x against the oracle (scale-relative, `tol`) and against ref64 (per element); a failure names every check that
    failed.  base: the input the output was added to (velocities): ref64 gives the change, compared with x - base above
    the float32 rounding of x."""
    failed = []
    try:
        assert_close(x, oracle, tol=tol, what=what)
    except AssertionError as e:
        failed.append(str(e))
    if base is not None:
        floor = floor + ref64.f32_spacing(x)
        x = np.asarray(x, np.float64) - np.asarray(base, np.float64)
    try:
        ref64.assert_per_element(x, ref, TAU, what + " (per element vs float64)", floor)
    except AssertionError as e:
        failed.append(str(e))
    assert not failed, " | ".join(failed)


def path_counts(s, path):
    """(counts, per-particle 'list usable' mask, staged-tile mask or None) of the list the sweeps walk"""
    from cpp_fluid_particles_b200 import capi
    if path.tile:
        cnt, _, win = s.tile_lists()
        cnt, win = cnt.cpu().numpy(), win.cpu().numpy()
        T = win[:, :, 1].sum(1)
        staged_tile = T <= capi.TILE_CAP
        staged = np.repeat(staged_tile, capi.TILE_PARTICLES)[:cnt.shape[0]]
        return cnt, staged, staged_tile
    cnt, _ = s.neighbor_list()
    return cnt.cpu().numpy(), np.ones(cnt.shape[0], bool), None


def run_sweeps(pkg, O, case: Case, path: Path, ratios=None):
    """Runs every sweep entry on `case` along `path`, asserts each output, and asserts that the path was taken.
    ratios (dict, optional) receives the largest |x - ref| / mag per output (the observed tau of DESIGN.md section 2)."""
    import torch
    if not torch.cuda.is_available():
        import pytest
        pytest.fail("pytest -m gpu needs a CUDA device: libsphk has no CPU fallback")
    from cpp_fluid_particles_b200 import capi, engine
    s = engine.SphkSystem(case.sc, step0=False, use_list=path.use_list, list_capacity=path.kmax)
    try:
        _run(torch, capi, O, s, case, path, ratios)
    finally:
        s.close()


def _run(torch, capi, O, s, case, path, ratios):
    p = case.sc.params
    s.set_option(capi.OPT_STAGED_LIST_BUILD, path.staged)
    s.set_option(capi.OPT_TILE, path.tile)
    s.set_use_list(path.use_list, path.skin)
    n = s.fluid.n
    mass = case_masses(case, n, p.m0)
    research = case.mass != "refresh"          # sphk_refresh alone sets the masses: the sweeps then walk the cells
    if case.mass != "refresh":
        s.fluid.mass.copy_(torch.from_numpy(mass))
    s.search_fluid()
    if case.mass == "refresh":
        s.fluid.mass.copy_(torch.from_numpy(mass))
        s.refresh()
    rcp = s.device_rcp(p.cell_length)
    st = s.state()
    g = O.grid(p.cell_size, p.cell_length, hash_rcp=rcp)
    A = O.SceneArrays(st["pos"], mass, st["cell_start"], st["posB"], st["massB"], st["cell_startB"], g, p.radius)
    P = ref64.Pairs(A)
    rng = np.random.default_rng(7)
    vel = (0.5 * np.sin(7.0 * st["pos"]) + 0.05 * rng.standard_normal((n, 3))).astype(F)
    zero = np.zeros_like(vel)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))   # noqa: E731

    def check(x, oracle, ref, what, **kw):
        if ratios is not None:
            xx = x if kw.get("base") is None else np.asarray(x, np.float64) - kw["base"]
            fl = ref64.f32_spacing(x) if kw.get("base") is not None else 0.0
            ratios[what] = max(ratios.get(what, 0.0), ref64.ratio(xx, ref, fl))
        _check(x, oracle, ref, what, **kw)

    def set_vel(v):
        s.fluid.vel.copy_(t(v))
        s.refresh()
        if research:       # refresh marks positions dirty; a new search re-validates the list on identical order
            s.search_fluid()

    # --- the path was taken ---
    if path.use_list and research:
        s.build_neighbor_list()
        cnt, staged, staged_tile = path_counts(s, path)
        kmax = path.kmax
        on_list = (cnt <= kmax) & staged
        if case.lattice_like:
            assert on_list.any(), "no particle walks the list"
        if path.kmax != 96 and case.lattice_like:
            assert ((cnt == kmax) & staged).any() and ((cnt == kmax + 1) & staged).any(), \
                f"capacity {kmax}: no particle with count == kmax and == kmax + 1 (counts {np.bincount(cnt)})"
            if kmax == 32:
                assert on_list.mean() >= 0.1 and (cnt > kmax).mean() >= 0.1, (on_list.mean(), (cnt > kmax).mean())
        if path.tile and case.lattice_like:
            assert staged_tile.any() and (~staged_tile).any(), "tile windows: want staged tiles and tiles beyond the cap"
        if not path.tile:
            # the list holds every pair within R of an in-grid particle; a skin list (radius R (1 + skin)) holds more
            inside = np.arange(n) < int(A.csF[p.ncells])
            within_r = np.bincount(P.iF, minlength=n) + np.bincount(P.iB, minlength=n)
            assert np.all(cnt[inside] >= within_r[inside]), "the list misses pairs within the support"
            if path.skin and within_r.sum() > 0:
                assert cnt[inside].sum() >= 1.2 * within_r[inside].sum(), "the skin list holds no more than the pairs within R"
        # (list_global: the staged and the global builder write the same list entry for entry -- compared by
        # test_tuned_list_builder_equals_simple_cell_walk -- so nothing in the results tells the two builders apart)

    # --- density + EOS ---
    s.density(); s.pressure()
    dens = O.density(A)
    ref_den = ref64.density(P)
    check(s.state()["density"], dens, ref_den, "density")
    if case.mass != "uniform":
        A0 = O.SceneArrays(A.posF, np.full(n, p.m0, F), A.csF, A.posB, A.massB, A.csB, g, p.radius)
        assert relerr(s.state()["density"], O.density(A0)) > 100 * TOL, "the masses must change the result"
    # (stiff raised so that the lattice, rho < rho0, still yields non-zero pressures for the force test)
    dhi = (dens * F(1.3)).astype(F)
    s.fluid.density.copy_(t(dhi))
    s.pressure()
    pres = O.pressure(dhi, p.rho0, p.stiff)
    assert_close(s.state()["pressure"], pres, what="pressure (Tait EOS)")
    bulk = n > 1000                            # (the small-n scenes are lines of particles far below rest density)
    assert pres.max() > 0 or not bulk
    s.fluid.pressure.copy_(t(pres))
    # pressure force
    set_vel(vel)
    s.pressure_force()
    v_ref = O.pressure_force(A, dhi, pres, vel, p.dt)
    x = s.state()["vel"]
    assert_close(x - vel, v_ref - vel, tol=2e-5 * case.force_scale, what="pressure force dv")
    check(x, v_ref, ref64.pressure_force_dv(P, dhi, pres, p.dt), "pressure force vel", base=vel, tol=TOL * case.force_scale)
    # viscosity
    set_vel(vel)
    s.viscosity()
    dv_ref = O.viscosity(A, vel, p.rho0, p.visc, p.dt)
    rv = ref64.viscosity_dv(P, vel, p.rho0, p.visc, p.dt)
    check(s.buffer3.cpu().numpy(), dv_ref, rv, "viscosity deltaV")
    check(s.state()["vel"], vel + dv_ref, rv, "viscosity vel", base=vel)
    # colour gradient + surface tension / air pressure (from rest: the change is not rounded into a velocity)
    s.color_grad()
    cg_ref = O.color_grad(A, p.rho0, p.rho_boundary)
    rcg = ref64.color_grad(P, p.rho0, p.rho_boundary)
    check(s.buffer3.cpu().numpy(), cg_ref, rcg, "colour gradient")
    set_vel(zero)
    s.buffer3.copy_(t(cg_ref))
    s.surface()
    v_ref = O.surface(A, cg_ref, zero, p.dt, p.rho0, p.surface_tension, p.air_pressure)
    rs = ref64.surface_dv(P, cg_ref, p.rho0, p.surface_tension, p.air_pressure, p.dt)
    check(s.state()["vel"], v_ref, rs, "surface dv", tol=2e-5, base=zero)
    # fused density + colour gradient
    s.fused_density_color_grad(False)
    check(s.state()["density"], dens, ref_den, "fused density (+colour gradient)")
    check(s.color_grad_buf.cpu().numpy(), cg_ref, rcg, "fused colour gradient (+density)")
    # DFSPH
    s.dfsph_density_alpha()
    d_ref, a_ref = O.dfsph_density_alpha(A)
    rd, ra = ref64.dfsph_density_alpha(P)
    check(s.state()["density"], d_ref, rd, "dfsph density")
    check(s.alpha.cpu().numpy(), a_ref, ra, "dfsph alpha")
    s.color_grad_buf.zero_()
    s.fused_density_color_grad(True)
    check(s.state()["density"], d_ref, rd, "fused dfsph density (+alpha, colour gradient)")
    check(s.alpha.cpu().numpy(), a_ref, ra, "fused dfsph alpha (+colour gradient)")
    check(s.color_grad_buf.cpu().numpy(), cg_ref, rcg, "fused colour gradient (+dfsph density, alpha)")
    set_vel(vel)
    s.alpha.copy_(t(a_ref)); s.fluid.density.copy_(t(d_ref))
    s.dfsph_div_error()
    e_ref, k_ref = O.dfsph_error(A, vel, d_ref, a_ref, p.dt, p.rho0, "div")
    re_, rk = ref64.dfsph_div_error(P, vel, d_ref, a_ref, p.dt, p.rho0, TAU)
    # the divergence sum cancels strongly; compare on the scale of its terms (sum_j m_j |v_ij . gradW_ij|)
    check(s.error.cpu().numpy(), e_ref, re_, "divergence error", tol=5e-5)
    check(s.kappa.cpu().numpy(), k_ref, rk, "divergence stiffness", tol=5e-5)
    for with_cg in (True, False):
        set_vel(vel)
        s.alpha.zero_(); s.error.zero_(); s.kappa.zero_(); s.color_grad_buf.zero_()
        s.fused_density_alpha_div_error(with_cg)
        what = "fused density/alpha/div error" + (" +colour gradient" if with_cg else "")
        dg, ag = s.state()["density"], s.alpha.cpu().numpy()
        check(dg, d_ref, rd, what + ": density")
        check(ag, a_ref, ra, what + ": alpha")
        if with_cg:
            check(s.color_grad_buf.cpu().numpy(), cg_ref, rcg, what + ": colour gradient")
        # the error's epilogue reads the density and alpha this particle has just formed
        fe, fk = ref64.dfsph_div_error(P, vel, dg, ag, p.dt, p.rho0, TAU)
        check(s.error.cpu().numpy(), e_ref, fe, what + ": error", tol=5e-5)
        check(s.kappa.cpu().numpy(), k_ref, fk, what + ": stiffness", tol=5e-5)
    set_vel(vel)
    s.kappa.copy_(t(k_ref))
    s.dfsph_div_correct()
    check(s.state()["vel"], O.dfsph_correct(A, k_ref, vel, 0.0), ref64.dfsph_correct_dv(P, k_ref), "divergence correct", base=vel)
    set_vel(vel)
    dens_hi = (d_ref * F(1.28)).astype(F)
    s.fluid.density.copy_(t(dens_hi))
    s.alpha.copy_(t(a_ref))                    # (the fused sweeps above left their own alpha there)
    s.warm.zero_()
    s.dfsph_den_error(True)
    e_ref, k_ref = O.dfsph_error(A, vel, dens_hi, a_ref, p.dt, p.rho0, "den")
    re_, rk = ref64.dfsph_den_error(P, vel, dens_hi, a_ref, p.dt, p.rho0)
    assert e_ref.max() > 0 or not bulk
    check(s.error.cpu().numpy(), e_ref, re_, "density error")
    check(s.kappa.cpu().numpy(), k_ref, rk, "density stiffness")
    check(s.warm.cpu().numpy(), k_ref, rk, "warm stiffness accumulate")
    set_vel(vel)                               # (a new search: the records mirror the stiffness copied in next)
    s.kappa.copy_(t(k_ref))
    s.dfsph_den_correct()
    check(s.state()["vel"], O.dfsph_correct(A, k_ref, vel, p.dt), ref64.dfsph_correct_dv(P, k_ref, p.dt), "density correct", base=vel)
    # abs-sum reduction (order unspecified in the reference: tolerance, not bit-exact)
    tot = s.reduce_abs_sum(s.error)
    assert abs(tot - float(np.abs(e_ref.astype(np.float64)).sum())) <= 1e-5 * max(1.0, float(np.abs(e_ref).sum()))
    # fused viscosity + surface: v_new = (v + deltaV) + a_surf * dt
    set_vel(vel)
    s.color_grad_buf.copy_(t(cg_ref))
    s.fused_viscosity_surface()
    check(s.buffer3.cpu().numpy(), dv_ref, rv, "fused viscosity deltaV (+surface)")
    v_ref = O.surface(A, cg_ref, vel + dv_ref, p.dt, p.rho0, p.surface_tension, p.air_pressure)
    both = ref64.R64(rv.value + rs.value, rv.mag + rs.mag, None if rs.alt is None else rv.value + rs.alt)
    check(s.state()["vel"], v_ref, both, "fused viscosity + surface vel", base=vel, floor=ref64.f32_spacing(vel + dv_ref))

    # --- PBD (rest density at the median density: about half the particles project, lambda != 0) ---
    p_pbd = dataclasses.replace(p, rho0=float(F(np.median(d_ref)))) if bulk else p
    s.p = p_pbd
    s.lam = torch.zeros(n, dtype=torch.float32, device=s.device)
    s.dpos = torch.zeros((n, 3), dtype=torch.float32, device=s.device)
    s.xsph_c, s.relaxation = 0.05, 0.75
    rho0 = p_pbd.rho0
    set_vel(vel)
    s.pbd_density_lambda()
    d_ref, l_ref = O.pbd_density_lambda(A, rho0, s.relaxation)
    rd, rl = ref64.pbd_density_lambda(P, rho0, s.relaxation)
    assert (l_ref != 0).sum() > n // 10 or not bulk
    check(s.state()["density"], d_ref, rd, "pbd density")
    check(s.lam.cpu().numpy(), l_ref, rl, "pbd lambda")
    pos0 = s.state()["pos"]
    set_vel(vel)
    s.lam.copy_(t(l_ref))
    s.pbd_delta_pos_apply()
    dp_ref = O.pbd_delta_pos(A, l_ref, rho0)
    check(s.dpos.cpu().numpy(), dp_ref, ref64.pbd_delta_pos(P, l_ref, rho0), "pbd delta pos")
    newpos = np.clip((pos0 + dp_ref).astype(F), 0.0, F(0.99) * F(p.space[0]))
    assert_close(s.state()["pos"], newpos, tol=1e-6, what="pbd applied positions")
    s.fluid.pos.copy_(t(pos0))
    set_vel(vel)
    s.pbd_xsph()
    rx = ref64.pbd_xsph_dv(P, vel, s.xsph_c, rho0)
    check(s.state()["vel"], O.pbd_xsph(A, vel, s.xsph_c, rho0), rx, "xsph", base=vel)
    set_vel(vel)
    s.buffer3.zero_()
    s.fused_pbd_xsph_color_grad()
    check(s.state()["vel"], O.pbd_xsph(A, vel, s.xsph_c, rho0), rx, "fused xsph (+colour gradient)", base=vel)
    check(s.buffer3.cpu().numpy(), O.color_grad(A, rho0, p.rho_boundary), ref64.color_grad(P, rho0, p.rho_boundary),
          "fused colour gradient (+xsph)")
    s.p = p

    # --- advect + clamp: push some particles through the walls ---
    big = vel.copy(); big[::5] *= 400.0
    set_vel(big)
    pos0 = s.state()["pos"]
    s.advect()
    p_ref, v_ref = O.advect(pos0, big, p.dt, p.space)
    st3 = s.state()
    assert_close(st3["pos"], p_ref, tol=1e-6, what="advect pos")
    assert np.array_equal(st3["vel"] == 0, v_ref == 0)
    assert_close(st3["vel"], v_ref, tol=1e-6, what="advect vel (clamped)")
    assert st3["pos"].min() >= 0.0 and st3["pos"].max() <= 0.99 * p.space[0] + 1e-7
