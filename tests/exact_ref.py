"""Exact references and forward-error bounds for the floating-point reductions, scans and groupby aggregations.

A float result is checked against the exactly rounded answer with a bound derived from the kernel, not a fixed tolerance:

    |got - exact| <= 2 * k * u * sum(|x_i|) + u_out * |exact|

u is the unit roundoff of the accumulator, u_out that of the output type, and k the longest chain of dependent additions
the kernel can form for that result. Any summation tree of depth k over the x_i is within k * u * sum(|x_i|) (1 + O(ku))
of the exact sum; the factor 2 covers the O(ku) term and the rounding of the exact reference itself. Each k below is
written next to the kernel constants it comes from, so a change to those constants shows up here.
"""
from __future__ import annotations

import itertools
import math
from fractions import Fraction

import numpy as np

U64 = 2.0 ** -53  # unit roundoff of float64
U32 = 2.0 ** -24  # unit roundoff of float32


def unit_roundoff(dtype) -> float:
    return U32 if np.dtype(dtype) == np.float32 else U64


# ---- k per kernel -------------------------------------------------------------------------------------------------

# reduce_kernel (scan_reduce.cu): 256 threads per block and 16 elements per thread at full occupancy, grid capped at 8 blocks
# per SM. A thread folds its elements in sequence (plus at most one of the unaligned head / tail), then a warp tree (5), thread
# 0 folds the 8 warp totals (7), the last block folds the partials 32-strided (ceil(grid / 32)) and by a warp tree (5), and the
# initial value is applied last (1).
REDUCE_THREADS, REDUCE_ELEMS_PER_THREAD, REDUCE_BLOCKS_PER_SM = 256, 16, 8


def reduce_grid(n: int, sms: int) -> int:
    return max(1, min(-(-n // (REDUCE_THREADS * REDUCE_ELEMS_PER_THREAD)), sms * REDUCE_BLOCKS_PER_SM))


def k_reduce(n: int, sms: int) -> int:
    grid = reduce_grid(n, sms)
    per_thread = -(-n // (REDUCE_THREADS * grid)) + 1
    return per_thread + 5 + 7 + -(-grid // 32) + 5 + 1


# scan_kernel (scan_reduce.cu): SC_THREADS = 512 (16 warps), V = 16 / sizeof(T) elements per vector, SC_K vectors per lane.
# In a tile: the vector's running sum (V), the warp's shuffle scan (5), the carry over the SC_K steps (SC_K), the prefix of the
# earlier warps (16) and two applications of it (2). The look-back folds up to SC_LB * 32 predecessor records by a per-lane
# chain (SC_LB) and a warp tree (5); a tile's inclusive prefix adds 2 to its predecessor's, so every earlier tile adds 2.
SC_WARPS, SC_LB = 16, 4


def scan_tile(itemsize: int) -> int:
    v = 16 // itemsize
    return 32 * v * (8 if itemsize == 8 else 4) * SC_WARPS


def k_scan(i: int, itemsize: int) -> int:
    v, sc_k = 16 // itemsize, (8 if itemsize == 8 else 4)
    return v + 5 + sc_k + SC_WARPS + 2 + SC_LB + 5 + 2 * (i // scan_tile(itemsize))


# segreduce_kernel (scan_reduce.cu): one warp per segment, lane l folds elements l, l + 32, ... (ceil(len / 32)), then a warp
# tree (5) and the initial value (1, counted in the 5 + 1 below with the store's conversion).
def k_segmented(length: int) -> int:
    return -(-length // 32) + 5


# groupby_kernel / pgb_agg_kernel (groupby.cu): every valid value is one atomic add, landing in any order, and the partitioned
# path merges partial sums made of the same values: no chain is longer than the group's valid count.
def k_hash_group(count: int) -> int:
    return max(count, 1)


# seg_tile_summary / seg_apply kernels (groupby.cu, SEG_TILE = 2048): row p of a group is the sequential running sum of its p + 1
# values plus one carry add per tile boundary crossed.
SEG_TILE = 2048


def k_grouped_scan(pos: int) -> int:
    return pos + 2 + pos // SEG_TILE


# ---- exact values -------------------------------------------------------------------------------------------------

def _scaled(x):
    """float values -> (Python ints, e) with x[i] == ints[i] * 2**e exactly."""
    x = np.asarray(x, np.float64)
    if len(x) == 0:
        return [], 0
    m, ex = np.frexp(x)
    mi = np.ldexp(m, 53).astype(np.int64)  # exact: |m| < 1, 53 bits
    ex = ex.astype(np.int64) - 53
    e = int(ex.min())
    return [int(a) << int(b - e) for a, b in zip(mi.tolist(), ex.tolist())], e


def _to_float(i: int, e: int) -> float:
    s = max(0, abs(i).bit_length() - 62)
    return math.ldexp(float(i >> s) if i >= 0 else -float((-i) >> s), e + s)


def exact_sum(x) -> float:
    return math.fsum(np.asarray(x, np.float64).tolist())


def abs_sum(x) -> float:
    return math.fsum(np.abs(np.asarray(x, np.float64)).tolist())


def special_sum(x):
    """Expected SUM of values that contain NaN or inf: NaN, +inf or -inf; None when every value is finite."""
    x = np.asarray(x, np.float64)
    if np.isnan(x).any() or (np.isposinf(x).any() and np.isneginf(x).any()):
        return math.nan
    if np.isposinf(x).any():
        return math.inf
    if np.isneginf(x).any():
        return -math.inf
    return None


def prefix_errors(got, x):
    """Exact |got[i] - sum(x[:i + 1])|, the exact prefix sums (rounded to float64) and the prefix sums of |x| (all finite)."""
    got = np.asarray(got, np.float64)
    ints, e = _scaled(np.concatenate([np.asarray(x, np.float64), got]))
    n = len(got)
    xs, gs = ints[:n], ints[n:]
    err, exact = np.empty(n), np.empty(n)
    for i, (p, g) in enumerate(zip(itertools.accumulate(xs), gs)):
        err[i] = _to_float(abs(g - p), e)
        exact[i] = _to_float(p, e)
    return err, exact, np.cumsum(np.abs(np.asarray(x, np.float64)))


def exact_m2(x) -> float:
    """sum((x - mean)^2) of finite values, exactly rounded."""
    ints, e = _scaled(x)
    n = len(ints)
    if n == 0:
        return 0.0
    s, q = sum(ints), sum(i * i for i in ints)
    m2 = Fraction(q * n - s * s, n) * Fraction(2) ** (2 * e)
    return float(m2)


# ---- bounds -------------------------------------------------------------------------------------------------------

def sum_bound(k: int, u: float, l1: float, exact: float, u_out: float) -> float:
    return 2 * k * u * l1 + u_out * abs(exact)


def mean_bound(k: int, u: float, l1: float, exact_sum_: float, count: int, u_out: float) -> float:
    """SUM bound (rounded in the accumulator), then one division rounded to the output type. A quotient in the subnormal
    range rounds to a multiple of the smallest subnormal, not relative to its size: that absolute step is added."""
    s = sum_bound(k, u, l1, exact_sum_, u) / count
    eta = 2.0 ** -1074 if u_out == U64 else 2.0 ** -149
    return s * (1 + u_out) + u_out * abs(exact_sum_ / count) + eta


def m2_bound(k: int, x) -> float:
    """Forward error of the reference's one-pass M2 = sumsq - sum^2 / n (m2_var_std.cu), with SUM and SUM_OF_SQUARES each
    accumulated in float64 along chains of length k (each square rounded once more)."""
    x = np.asarray(x, np.float64)
    n = len(x)
    s, q = abs(exact_sum(x)), math.fsum((x * x).tolist())
    es = 2 * k * U64 * abs_sum(x)
    eq = (2 * k + 1) * U64 * q
    s_hi = s + es
    d = s_hi * s_hi / n
    return eq + (2 * s * es + es * es) / n + 3 * U64 * d + U64 * (q + eq + d)


def var_std_bounds(k: int, x, ddof: int):
    """(exact VAR, its bound, exact STD, its bound) from the M2 bound: one division, then one square root."""
    n = len(x)
    m2 = exact_m2(x)
    var = m2 / (n - ddof)
    bv = m2_bound(k, x) / (n - ddof) + 2 * U64 * abs(var)
    std = math.sqrt(var)
    bs = max(math.sqrt(var + bv) - std, std - math.sqrt(max(var - bv, 0.0))) + 2 * U64 * std
    return var, bv, std, bs


def two_pass_bounds(k: int, x, delta: float, ddof: int):
    """Forward error of the sort path's two-pass M2 / VARIANCE / STD (group_m2.cu, group_std.cu) over finite x, with the group
    mean computed to within delta and the per-row terms summed along chains of length k.

    sum((x - m)^2) = M2 + n (m - mean)^2 exactly for any m, so the computed mean adds at most n delta^2. Each term is rounded
    by the difference and the square (and the division by n - ddof for VARIANCE), and the sum of those non-negative terms adds
    k u relative; (2k + 3) u covers both with room for the second-order terms.
    -> (M2, its bound, VAR, its bound, STD, its bound); VAR / STD are None when n <= ddof."""
    n = len(x)
    m2 = exact_m2(x)
    shift = n * delta * delta
    bm = shift + (2 * k + 3) * U64 * (m2 + shift) + U64 * m2
    if n - ddof <= 0:
        return m2, bm, None, None, None, None
    var = m2 / (n - ddof)
    bv = (shift + (2 * k + 4) * U64 * (m2 + shift)) / (n - ddof) + U64 * var
    std = math.sqrt(var)
    bs = max(math.sqrt(var + bv) - std, std - math.sqrt(max(var - bv, 0.0))) + 2 * U64 * std
    return m2, bm, var, bv, std, bs


def check(got, exact, bound, what=""):
    """got within bound of exact; NaN / inf results are compared as values."""
    got, exact = float(got), float(exact)
    if math.isnan(exact) or math.isinf(exact):
        assert (math.isnan(got) and math.isnan(exact)) or got == exact, f"{what}: got {got!r}, expected {exact!r}"
        return
    assert math.isfinite(got) and abs(got - exact) <= bound, \
        f"{what}: got {got!r}, exact {exact!r}, error {abs(got - exact):.3e} > bound {bound:.3e}"
