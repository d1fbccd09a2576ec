"""The host emulations of tests/reduction_ref.py (DESIGN.md section 2.7) against independent restatements: a scalar loop over
the kernels' threads for the fixed-shape sum, math.fsum for its error bound, and the reference's two while loops for the
loop model.  No GPU."""
import math

import numpy as np
import pytest

import reduction_ref as RD

F = np.float32


def _scalar_tree(x):
    """k_abs_sum_partial + k_abs_sum_final written out per thread, one float32 add at a time"""
    a = [F(0) if abs(F(v)) < F(RD.TINY) else abs(F(v)) for v in np.asarray(x, F).ravel()]
    n = len(a)
    g = min(max((n + 2047) // 2048, 1), 1024)

    def block(values):                 # values[t]: thread t's sum; warp butterflies, then the 8 warp sums
        s = list(values)
        for o in (16, 8, 4, 2, 1):
            s = [F(s[t] + s[(t & ~31) | ((t & 31) ^ o)]) for t in range(256)]
        w = [s[32 * k] for k in range(8)]
        for o in (4, 2, 1):
            w = [F(w[t] + w[t ^ o]) for t in range(8)]
        return w[0]

    part = []
    for b in range(g):
        th = []
        for t in range(256):
            s, i = F(0), b * 256 + t
            while i < n:
                s = F(s + a[i])
                i += g * 256
            th.append(s)
        part.append(block(th))
    th = []
    for t in range(256):
        s, i = F(0), t
        while i < g:
            s = F(s + part[i])
            i += 256
        th.append(s)
    return block(th)


def _mixed(n, seed, spread=20):
    """seeded mixed-sign values over 2^+-spread"""
    rng = np.random.default_rng(seed)
    return (rng.choice([-1.0, 1.0], n) * np.exp2(rng.uniform(-spread, spread, n))).astype(F)


@pytest.mark.parametrize("n", [1, 7, 31, 255, 256, 257, 2047, 2048, 2049, 5000, 3 * 2048 + 5])
def test_tree_matches_a_scalar_loop_of_the_same_shape(n):
    x = _mixed(n, n)
    assert RD.tree_abs_sum(x).view(np.uint32) == _scalar_tree(x).view(np.uint32)


def test_tree_matches_a_scalar_loop_past_256_partials():
    """the final stage's second pass: 257 partials (n = 257 * 2048).  The partials are formed the vectorised way (checked
    against the scalar loop above at smaller n) and the final stage against a scalar loop of its own"""
    x = _mixed(257 * 2048, 5)
    p = RD.partials(x)
    assert p.size == 257
    s = [F(0)] * 256
    for i, v in enumerate(p):
        s[i % 256] = F(s[i % 256] + v)
    th = np.array(s, F).reshape(8, 32)
    for o in (16, 8, 4, 2, 1):
        th = th + th[:, np.arange(32) ^ o]
    w = th[:, 0]
    for o in (4, 2, 1):
        w = w + w[np.arange(8) ^ o]
    assert RD.final(p).view(np.uint32) == F(w[0]).view(np.uint32)
    # dropping the partials past 256 changes the sum
    assert RD.final(p[:256]) != RD.final(p)


def test_subnormals_are_flushed():
    tiny = np.array([1e-40, -1e-39, 2.0 ** -127, 2.0 ** -126], F)
    assert RD.tree_abs_sum(tiny) == F(2.0 ** -126)
    assert RD.tree_abs_sum(np.zeros(3, F)) == 0


def test_blocks_follow_the_launch():
    assert [RD.blocks(n) for n in (0, 1, 2048, 2049, 1024 * 2048, 1024 * 2048 + 1, 10 ** 8)] == [1, 1, 1, 2, 1024, 1024, 1024]


@pytest.mark.parametrize("n,spread", [(1, 20), (1000, 20), (2049, 3), (256 * 2048 + 1, 20), (1024 * 2048 + 1, 20),
                                      (5_000_000, 20), (5_000_000, 1)])
def test_tree_is_within_its_bound_of_fsum(n, spread):
    x = _mixed(n, 11 + n, spread)
    got = float(RD.tree_abs_sum(x))
    ref = math.fsum(np.abs(x.astype(np.float64)).tolist())
    err = abs(got - ref)
    b = RD.bound(x)
    assert err <= b, f"n = {n}: |tree - fsum| = {err:.3e} > bound {b:.3e}"
    # the bound is not vacuous: a few hundred ulps of the sum at most
    assert b <= 64 * RD.depth(n) * RD.U * ref


# ---- the loop model ---------------------------------------------------------------------------------------------------------
def _reference_divergence(thr, totals, max_iter):
    """DFSPHSolver::correctDivergenceError's loop, DFSPHSolver.cu:347-360 (the sweeps left out)"""
    total, it = RD.FLT_MAX, 0
    while (it < 1 or total > thr) and it < max_iter:
        it += 1
        total = F(totals[it - 1])
    return it, total


def _reference_density(thr, totals, max_iter):
    """DFSPHSolver::project's loop, DFSPHSolver.cu:187-207"""
    total, it = RD.FLT_MAX, 0
    while (it < 2 or total > thr) and it < max_iter:
        it += 1
        if it >= 2:
            total = F(totals[it - 1])
    return it, total


def _same(a, b):
    return a[0] == b[0] and a[1].view(np.uint32) == b[1].view(np.uint32)


T = RD.loop_threshold(1e-3, 2 ** 21, 1.0)
UP, DOWN = np.nextafter(T, F(np.inf)), np.nextafter(T, F(0))
SEQUENCES = {
    "converges at 3": [9 * T, 5 * T, DOWN, 0.5 * T, 0.1 * T],
    "exactly the threshold": [9 * T, 2 * T, T, 0.5 * T],
    "one ulp above": [9 * T, 2 * T, UP, T, 0.5 * T],
    "one ulp below": [9 * T, 2 * T, DOWN, 0.5 * T],
    "huge first": [RD.FLT_MAX, 0.1 * T, 0.1 * T, 0.1 * T],
    "small first": [0.1 * T, 0.1 * T, 5 * T, 0.1 * T],
    "nan": [9 * T, np.nan, 9 * T, 9 * T, 9 * T],
    "inf": [np.inf, np.inf, 0.0, 0.0],
    "never": [9 * T] * 25,
}


@pytest.mark.parametrize("name", sorted(SEQUENCES))
@pytest.mark.parametrize("max_iter", [0, 1, 2, 3, 20])
def test_loop_model_is_the_reference_loops(name, max_iter):
    totals = [F(t) for t in SEQUENCES[name]] + [F(9 * T)] * 25
    assert _same(RD.loop_model(1, max_iter, T, 1, totals), _reference_divergence(T, totals, max_iter))
    assert _same(RD.loop_model(2, max_iter, T, 2, totals), _reference_density(T, totals, max_iter))


def test_loop_model_edges():
    assert RD.loop_model(1, 20, T, 1, [T, 0, 0])[0] == 1, "a total equal to the threshold stops the loop"
    assert RD.loop_model(1, 20, T, 1, [UP, DOWN, 0])[0] == 2
    assert RD.loop_model(2, 20, T, 2, [RD.FLT_MAX, 0.0, 0.0])[0] == 2, "the first error is not read from iteration 2 on"
    assert RD.loop_model(2, 20, T, 2, [0.0, 5 * T, 0.0, 0.0])[0] == 3, "min_iter = 2 runs on past a small first total"
    it, tot = RD.loop_model(1, 20, T, 1, [9 * T, np.nan, 0.0])
    assert it == 2 and np.isnan(tot), "a NaN total ends the loop"
    assert RD.loop_model(1, 0, T, 1, [])[0] == 0
    assert RD.loop_model(0, 5, RD.FLT_MAX, 1, [0.0])[0] == 0, "FLT_MAX > FLT_MAX is false: no iteration without min_iter"


def test_loop_threshold_is_formed_in_float32():
    # 1e-3 * 2097152 * 1 in float32 differs from the double product: the class layer's (thr * num) * rho0 order
    t = RD.loop_threshold(1e-3, 2 ** 21 + 2049, 1.0)
    assert t.dtype == np.float32
    assert float(t) != 1e-3 * (2 ** 21 + 2049)
    assert RD.loop_threshold(1e-3, 16777217, 1.0) == RD.loop_threshold(1e-3, 16777216, 1.0), "num is rounded to float"
