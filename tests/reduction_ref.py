"""Exact host emulations of the engine's fixed-shape reductions and of the adaptive DFSPH loop test (DESIGN.md section 2.7).
numpy only.

tree_abs_sum is sphk_reduce_abs_sum (k_abs_sum_partial / k_abs_sum_final) and the error sum of the device loops
(k_loop_partial / k_loop_finish) operation for operation in float32: float adds are not reassociated and round to nearest
even on both sides, so the GPU result must match it bit for bit.  The library is built with -use_fast_math, whose adds flush
subnormal operands to zero; the inputs are flushed the same way (sums of non-negative normal numbers never fall below 2^-126).

loop_model restates k_loop_begin / k_loop_finish, which follow DFSPHSolver.cu:187,205-207,347,360 of the reference."""
import math

import numpy as np

F = np.float32
THREADS = 256                    # threads per block of both stages
PER_THREAD = 8                   # elements per thread before the block count grows
MAX_BLOCKS = 1024                # partials, at most (the size of the context's partial array)
FLT_MAX = F(np.finfo(np.float32).max)
U = 2.0 ** -24                   # unit roundoff of float32
TINY = 2.0 ** -126               # smallest normal float32


def blocks(n: int) -> int:
    """first-stage grid of sphk_reduce_abs_sum / sphk_loop_next: clamp(ceil(n / 2048), 1, 1024)"""
    return min(max((n + THREADS * PER_THREAD - 1) // (THREADS * PER_THREAD), 1), MAX_BLOCKS)


def flushed_abs(x) -> np.ndarray:
    """|x| in float32 with subnormals flushed to zero (FTZ adds); NaN and inf pass through"""
    a = np.abs(np.asarray(x, F).ravel())
    a[a < F(TINY)] = F(0)
    return a


def _thread_sums(a: np.ndarray, threads: int) -> np.ndarray:
    """thread j of `threads` adds a[j], a[j + threads], ... in that order, starting from 0 (grid-stride loop)"""
    rows = max(1, -(-a.size // threads))
    pad = np.zeros(rows * threads, F)
    pad[:a.size] = a
    s = np.zeros(threads, F)
    for r in pad.reshape(rows, threads):       # adding the padding's zeros is exact
        s = s + r
    return s


def _butterfly(s: np.ndarray, width: int) -> np.ndarray:
    """s += shfl_xor(s, o) for o = width/2 ... 1 along the last axis; lane 0's value"""
    lane = np.arange(width)
    o = width // 2
    while o > 0:
        s = s + s[..., lane ^ o]
        o >>= 1
    return s[..., 0]


def _block_sum(s: np.ndarray) -> np.ndarray:
    """(B, 256) thread values -> (B,) block totals: warp butterfly 16..1, then an 8-lane butterfly 4..1 over the warp sums"""
    warps = _butterfly(s.reshape(s.shape[0], THREADS // 32, 32), 32)
    return _butterfly(warps, THREADS // 32)


def partials(x) -> np.ndarray:
    """the first stage: one float32 partial per block"""
    a = flushed_abs(x)
    g = blocks(a.size)
    return _block_sum(_thread_sums(a, g * THREADS).reshape(g, THREADS))


def final(p) -> F:
    """the second stage: one block of 256 threads over the partials (thread t adds p[t], p[t + 256], ...)"""
    return F(_block_sum(_thread_sums(np.asarray(p, F), THREADS).reshape(1, THREADS))[0])


def tree_abs_sum(x) -> F:
    """sum |x_i| in the engine's fixed shape, bit for bit"""
    return final(partials(x))


def depth(n: int) -> int:
    """the most float adds any element passes through: its thread's grid-stride sum, the two butterflies of the first
    stage, its final-stage thread's sum and the two butterflies again"""
    g = blocks(n)
    return -(-max(n, 1) // (g * THREADS)) + 8 + -(-g // THREADS) + 8


def exact_abs_sum(x) -> float:
    """math.fsum of the flushed |x_i|: the exactly rounded sum"""
    return math.fsum(flushed_abs(x).astype(np.float64).tolist())


def bound(x) -> float:
    """|tree_abs_sum(x) - exact_abs_sum(x)| <= gamma_k sum |x_i| (k = depth) for summands >= 0 (every partial sum is
    <= sum |x_i|), and the terms FTZ dropped"""
    a = flushed_abs(x).astype(np.float64)
    k = depth(a.size)
    return k * U / (1.0 - k * U) * float(a.sum()) + a.size * TINY


def loop_threshold(thr, num, rho0) -> F:
    """errorThreshold * num * rho0 as the class layer forms it: float32, left to right, num rounded to float"""
    return F(F(F(thr) * F(num)) * F(rho0))


def loop_model(min_iter: int, max_iter: int, threshold, reduce_from: int, totals):
    """(iterations, last total) of a device loop: total starts at FLT_MAX; iteration k (1-based) reads totals[k - 1] when
    k >= reduce_from; the loop runs on while (iters < min_iter || total > threshold) && iters < max_iter.  A NaN total
    compares false, which ends the loop (once min_iter is reached), as in the reference."""
    thr = F(threshold)
    iters, total = 0, FLT_MAX

    def active():
        return (iters < min_iter or bool(total > thr)) and iters < max_iter

    while active():
        iters += 1
        if iters >= reduce_from:
            total = F(totals[iters - 1])
    return iters, total
