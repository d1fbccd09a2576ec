"""DFSPH chunk activity (DESIGN.md section 4.4): skipped sweeps leave every output bit-identical.

The reference run is the same engine with one uncounted launch announced (sphk_add_launches) before every DFSPH sweep: any launch
the library does not know to be harmless drops the chunk bits and the error sweeps' reuse token, so there every sweep walks
all its neighbours.  Compared bit for bit over the free fall (every chunk quiet), the impact and the partly active state after
it (200k scene, steps 1-45), and with a scalar write between an error sweep and its correct sweep."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pkgload  # noqa: E402

pkg = pkgload.load()
from cpp_fluid_particles_b200 import engine  # noqa: E402

pytestmark = pytest.mark.gpu

SWEEPS = ("fused_density_alpha_div_error", "dfsph_div_error", "dfsph_den_error", "dfsph_div_correct", "dfsph_den_correct")


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


def _same(a, b, what):
    for f in ("pos", "vel", "density"):
        x, y = a[f], b[f]
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), f"{what}: {f} differs in {np.sum(x.view(np.int32) != y.view(np.int32))} words"


def test_trajectory_bit_identical_through_impact():
    fast, ref = _system(False), _system(True)
    quiet_seen, mixed_seen = False, False
    for step in range(1, 46):
        fast.step(); ref.step()
        k = _bits(fast.kappa[: fast.n_total()])
        quiet = k == np.int32(-2**31)
        quiet_seen |= bool(quiet.all())
        mixed_seen |= bool(quiet.any() and not quiet.all())
        if step in (5, 20, 28, 32, 38, 45):
            _same(fast.state(), ref.state(), f"step {step}")
            assert np.array_equal(k, _bits(ref.kappa[: ref.n_total()])), f"step {step}: kappa"
            assert np.array_equal(_bits(fast.warm[: fast.n_total()]), _bits(ref.warm[: ref.n_total()])), f"step {step}: warm"
            assert np.array_equal(_bits(fast.error[: fast.n_total()]), _bits(ref.error[: ref.n_total()])), f"step {step}: error"
    assert quiet_seen and mixed_seen, "the run must cover an all-quiet and a partly active pressure solve"
    fast.close(); ref.close()


def test_scalar_write_between_error_and_correct():
    """A PBD lambda sweep overwrites the record scalar after a quiet error sweep: the correct sweep must re-mirror kappa and
    may not trust chunk bits that described the overwritten scalar."""
    a, b = _system(False, "mini"), _system(True, "mini")
    for s in (a, b):
        s.step()
        s.dfsph_div_error()
        lam = torch.full_like(s.kappa, 1.0e-3)
        s.L.sphk_pbd_density_lambda(s.ctx, s._s(), engine._ptr(lam), engine.C.c_float(s.p.rho0), engine.C.c_float(1.0))
        s.dfsph_div_correct()
        s.dfsph_div_error()
        s.dfsph_div_correct()
    torch.cuda.synchronize()
    _same(a.state(), b.state(), "lambda between error and correct")
    a.close(); b.close()
