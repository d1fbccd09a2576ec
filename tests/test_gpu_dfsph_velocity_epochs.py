"""DFSPH velocity epochs (DESIGN.md section 4.4): a quiet chunk's correct-sweep epilogue runs once per stretch of correct
sweeps, and every output stays bit-identical.

The reference is the engine with one uncounted launch announced (sphk_add_launches) before every DFSPH sweep: that drops the
chunk bits, the error sweeps' reuse token and the velocity epoch, so there every correct sweep walks all its neighbours and
writes every velocity.  The cases put -0 components into the fluid velocities, which the walk turns into +0 and a quiet chunk
must turn into +0 too -- in both the API array and the records -- and end an epoch by a copy over the velocities and by a
velocity launch between two correct sweeps.  The class layer's captured step graph runs through the impact against the
reference, so marks left by an earlier replay are exercised as well."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import capi, engine  # noqa: E402

pytestmark = pytest.mark.gpu

SWEEPS = ("fused_density_alpha_div_error", "dfsph_div_error", "dfsph_den_error", "dfsph_div_correct", "dfsph_den_correct")
NEG0 = np.int32(-2**31)


def _system(defeat: bool, scene="200k"):
    s = engine.SphkSystem(pkg.scene.benchmark_scene(scene, "dfsph"), device=torch.device("cuda:0"))
    if defeat:
        for name in SWEEPS:
            inner = getattr(s, name)

            def wrapped(*a, _inner=inner, **k):
                s.L.sphk_add_launches(s.ctx, 1)
                return _inner(*a, **k)
            setattr(s, name, wrapped)
    return s


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu().numpy()


def _vel_bits(s):
    return _bits(s.fluid.vel[: s.n_total()])


def _same_state(a, b, what):
    for f in ("pos", "vel", "density"):
        x, y = a[f], b[f]
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), f"{what}: {f} differs in {np.sum(x.view(np.int32) != y.view(np.int32))} words"


def _all_quiet(s):
    k = _bits(s.kappa[: s.n_total()])
    n32 = k.size // 32 * 32
    return bool((k[:n32] == NEG0).all())


def _snapshot_before(s, name, store):
    """records the fluid velocities each time s.<name> is about to run"""
    inner = getattr(s, name)

    def wrapped(*a, **k):
        store.append(_vel_bits(s))
        return inner(*a, **k)
    setattr(s, name, wrapped)


def _negate_zero_x(v):
    """vx = -0 wherever |vx| < 1e-4 (in free fall the block barely moves sideways); returns the particles hit"""
    hit = v[:, 0].abs() < 1e-4
    v[:, 0] = torch.where(hit, torch.full_like(v[:, 0], -0.0), v[:, 0])
    torch.cuda.synchronize()
    return hit.cpu().numpy()


def _quiet_chunks(kappa_bits):
    n32 = kappa_bits.size // 32 * 32
    return (kappa_bits[:n32].reshape(-1, 32) == NEG0).all(axis=1)


def test_negative_zero_velocities_of_quiet_chunks():
    """-0 components in the API velocities before a free-fall step: the search carries them into the records, the step's first
    correct sweep finds every chunk quiet and must turn them into +0 in both arrays, as the walk does."""
    fast, ref = _system(False), _system(True)
    for s in (fast, ref):
        for _ in range(3):
            s.step()
    assert _all_quiet(fast), "the case needs a free-fall step: every chunk quiet"
    snaps = {id(fast): ([], []), id(ref): ([], [])}
    for s in (fast, ref):
        hit = _negate_zero_x(s.fluid.vel[: s.n_total()])
        after_div, after_den = snaps[id(s)]
        _snapshot_before(s, "gravity", after_div)      # the divergence solve's velocities
        _snapshot_before(s, "advect", after_den)       # the density solve's velocities
        if s is fast:
            kap = []
            inner = s.dfsph_div_correct
            s.dfsph_div_correct = lambda *a, _i=inner, _s=s, **k: (kap.append(_bits(_s.kappa[: _s.n_total()])), _i(*a, **k))[1]
        s.step()
    quiet = _quiet_chunks(kap[0])
    hit_chunks = hit[: quiet.size * 32].reshape(-1, 32).any(axis=1)
    assert (quiet & hit_chunks).sum() >= 100, f"-0 in {hit.sum()} particles, {(quiet & hit_chunks).sum()} of them in quiet chunks"
    for k in (0, 1):
        a, b = snaps[id(fast)][k][0], snaps[id(ref)][k][0]
        assert not (b[:, 0] == NEG0).any(), "the walk turns -0 + 0 into +0"
        assert np.array_equal(a, b), f"solve {k}: velocities differ in {np.sum(a != b)} words"
    _same_state(fast.state(), ref.state(), "after the step")
    for s in (fast, ref):                               # the records' velocities reach the API arrays through the next step
        s.step()
    _same_state(fast.state(), ref.state(), "one step later")
    fast.close(); ref.close()


@pytest.mark.parametrize("between", ["copy", "gravity"])
def test_velocity_write_between_correct_sweeps(between):
    """Between two quiet correct sweeps of the divergence solve, a copy over the velocities (-0 components, not a launch) or a
    gravity launch: either ends the epoch, so the next correct sweep may not trust the marks the first one left."""
    fast, ref = _system(False), _system(True)
    for s in (fast, ref):
        for _ in range(3):
            s.step()
    assert _all_quiet(fast)
    after = {}
    for s in (fast, ref):
        inner = s.dfsph_div_correct
        calls = [0]
        after[id(s)] = []

        def wrapped(*a, _s=s, _inner=inner, _calls=calls, **k):
            _calls[0] += 1
            if _calls[0] == 2:
                if between == "copy":
                    v = _s.fluid.vel.clone()
                    _negate_zero_x(v)
                    _s.copy(_s.fluid.vel, v)
                else:
                    _s.gravity()
            r = _inner(*a, **k)
            after[id(_s)].append(_vel_bits(_s))
            return r
        s.dfsph_div_correct = wrapped
        s.step()
    assert _all_quiet(fast)
    a, b = after[id(fast)], after[id(ref)]
    assert len(a) == len(b) >= 2
    if between == "copy":
        assert not (b[1][:, 0] == NEG0).any()
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f"correct sweep {k + 1}: velocities differ in {np.sum(x != y)} words"
    for s in (fast, ref):
        s.step()
    _same_state(fast.state(), ref.state(), f"{between}: one step later")
    fast.close(); ref.close()


def test_class_layer_graph_through_impact():
    """The C++ class layer (captured step graph from its third step on) against the reference engine, steps 1-45 of the 200k
    scene: free fall, impact, partly active.  A replay repeats the trust flags of the captured sweeps; the first sweep of every
    epoch rewrites all marks before any is trusted, so marks left by the previous replay never count."""
    sc = pkg.scene.benchmark_scene("200k", "dfsph")
    app = capi.SphApp(sc)
    ref = _system(True)
    replayed = False
    for step in range(1, 46):
        app.step(); ref.step()
        replayed |= app.step_graph_active()
        if step in (5, 20, 28, 32, 38, 45):
            a, b = app.download(), ref.state()
            for f in ("pos", "vel", "density"):
                x, y = a[f].view(np.int32), b[f].view(np.int32)
                assert np.array_equal(x, y), f"step {step}: {f} differs in {np.sum(x != y)} words"
    assert replayed, "the class layer must replay its step graph"
    app.close(); ref.close()
