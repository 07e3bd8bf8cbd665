"""The aggregation reference (tests/aggs_reference.py) against literal restatements of the reference's collector loops
(MaxCollectorManager.java:117-121 and its Min / Sum twins, the terms collectors' per-value counts), on small arrays
holding NaN, +-inf, +-0, subnormals and +-Double.MAX_VALUE; and its decoders against the sortable encodings. CPU only."""
import math

import numpy as np
import pytest

import aggs_reference as ar
from nrtsearch_b200.search import double_to_sortable_long, float_to_sortable_int

M = ar.DBL_MAX
F32_MAX = float(np.finfo(np.float32).max)
SPECIAL = [math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324, -5e-324, 1e-310, -2.5e-315, M, -M, 1.5, -2.25, 3.0, 1e300,
           -1e300, 7e-300]


def java_max(vals):
    m = -M   # UNSET_VALUE
    for v in vals:
        if v > m:
            m = v
    return m


def java_min(vals):
    m = M
    for v in vals:
        if v < m:
            m = v
    return m


def java_sum(vals):
    s = 0.0
    for v in vals:
        s += v
    return s


def java_terms(vals, size, order_desc):
    counts = {}
    for v in vals:
        counts[int(v)] = counts.get(int(v), 0) + 1
    items = sorted(counts.items(), key=lambda kv: ((-kv[1] if order_desc else kv[1]), kv[0]))
    shown = items[:size]
    return shown, len(counts), sum(counts.values()) - sum(c for _, c in shown)


@pytest.mark.parametrize("seed", range(6))
def test_min_max_sum_match_the_collector_loops(seed):
    rng = np.random.default_rng(seed)
    for trial in range(400):
        n = int(rng.integers(0, 13))
        vals = [SPECIAL[i] for i in rng.integers(0, len(SPECIAL), n)]
        if trial % 3 == 0:
            vals += rng.normal(0, 1e6, int(rng.integers(0, 6))).tolist()
        mx, mn = ar.max_value(vals), ar.min_value(vals)
        assert mx == java_max(vals) and mn == java_min(vals), vals   # (zeros compare equal: the sign follows the order)
        assert not math.isnan(mx) and not math.isnan(mn)
        for _ in range(4):   # every summation order passes, as the device's atomics add in any order
            perm = [vals[i] for i in rng.permutation(len(vals))]
            assert ar.sum_ok(java_sum(perm), vals), (perm, ar.sum_value(vals))


def test_min_max_unset_side_and_nan():
    assert ar.max_value([]) == -M and ar.min_value([]) == M
    assert ar.max_value([math.nan]) == -M and ar.min_value([math.nan]) == M
    assert ar.max_value([-math.inf]) == -M and ar.min_value([math.inf]) == M
    assert ar.max_value([math.inf, math.nan]) == math.inf and ar.min_value([-math.inf, math.nan]) == -math.inf
    assert ar.max_value([math.nan, -math.inf, -5.0]) == -5.0 and ar.min_value([math.nan, math.inf, 5.0]) == 5.0
    assert ar.max_value([-M]) == -M and ar.min_value([M]) == M
    assert ar.max_value([-0.0]) == 0.0 and ar.min_value([5e-324, -5e-324]) == -5e-324


def test_sum_non_finite_and_bound():
    assert math.isnan(ar.sum_value([1.0, math.nan])[0]) and math.isnan(ar.sum_value([math.inf, -math.inf])[0])
    assert ar.sum_value([math.inf, M, 1.0]) == (math.inf, 0.0) and ar.sum_value([-math.inf, 1.0]) == (-math.inf, 0.0)
    assert ar.sum_value([]) == (0.0, 0.0)
    assert ar.sum_value([M, M, -M])[0] is None                   # an order that overflows exists
    assert ar.sum_ok(math.inf, [M, M, -M]) and ar.sum_ok(M, [M, M, -M]) and not ar.sum_ok(math.nan, [M, M, -M])
    assert ar.sum_ok(math.nan, [math.inf, -M, -M]) and ar.sum_ok(math.inf, [math.inf, -M, -M])   # -M - M overflows first
    exp, bound = ar.sum_value([1e16, 1.0, -1e16])                  # cancellation: the bound is absolute, not relative
    assert exp == 1.0 and bound == 3 * 2.0**-53 * (2e16 + 1.0)
    assert ar.sum_ok(java_sum([1e16, 1.0, -1e16]), [1e16, 1.0, -1e16])   # 0.0, an error of 100 % of the result
    assert not ar.sum_ok(1.0 + 2 * bound, [1e16, 1.0, -1e16]) and not ar.sum_ok(-math.inf, [math.inf, 1.0])
    vals = list(range(-1000, 2001))                               # integers below 2^53: every order is exact
    assert ar.sum_value(vals)[0] == java_sum(vals) == float(sum(vals))


@pytest.mark.parametrize("seed", range(4))
def test_terms_match_a_counting_loop(seed):
    rng = np.random.default_rng(100 + seed)
    for _ in range(200):
        n_distinct = int(rng.integers(1, 40))
        pool = rng.choice(np.arange(-2**62, 2**62, 2**55, dtype=np.int64), n_distinct, replace=False)
        pool[0] = np.iinfo(np.int64).min if seed % 2 else np.iinfo(np.int64).max
        vals = pool[rng.integers(0, n_distinct, int(rng.integers(0, 120)))]
        for size in (1, 3, 7, 64):
            for desc in (True, False):
                got = ar.terms(vals, size, desc)
                shown, total, other = java_terms(vals.tolist(), size, desc)
                n = len(shown)
                assert got["n"] == n and got["total_buckets"] == total and got["other_counts"] == other
                assert got["keys"][:n].tolist() == [k for k, _ in shown] and got["counts"][:n].tolist() == [c for _, c in shown]
                assert not got["keys"][n:].any() and not got["counts"][n:].any()
    got = ar.terms(np.zeros(0, np.int64), 5)
    assert got["n"] == 0 and got["total_buckets"] == 0 and got["other_counts"] == 0
    got = ar.terms_from_counts([9, -4, 7, 3], [2, 5, 2, 0], 2)     # ties go to the smaller value; empty buckets vanish
    assert got["keys"].tolist() == [-4, 7] and got["total_buckets"] == 3 and got["other_counts"] == 2


def test_decoders_invert_the_sortable_encodings():
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 2**32, 300, dtype=np.uint64).astype(np.uint32).view(np.float32)
    floats = np.concatenate([np.array([math.nan, math.inf, -math.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, F32_MAX, -F32_MAX], np.float32),
                             rng.normal(0, 1e3, 300).astype(np.float32), bits[~np.isnan(bits)]])   # (Lucene stores the canonical NaN)
    stored = np.array([float_to_sortable_int(float(f)) for f in floats], np.int64)
    got = ar.decode_float(stored)
    assert np.array_equal(got.astype(np.float32).view(np.uint32), floats.view(np.uint32))   # bit for bit
    assert got.dtype == np.float64 and np.array_equal(got[~np.isnan(got)], floats[~np.isnan(floats)].astype(np.float64))
    doubles = np.concatenate([np.array([math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324, -5e-324, 1e-310, M, -M]),
                              rng.normal(0, 1e100, 300), rng.integers(-2**63, 2**63 - 1, 300, dtype=np.int64).view(np.float64)])
    stored = np.array([double_to_sortable_long(float(d)) for d in doubles], np.int64)
    assert np.array_equal(ar.decode_double(stored).view(np.int64), doubles.view(np.int64))
    # the stored domain orders as the numbers do (NaN aside), which the terms keys and range queries rely on
    ok = ~np.isnan(doubles)
    order = np.argsort(stored[ok], kind="stable")
    assert (np.diff(doubles[ok][order]) >= 0).all()
    assert np.array_equal(ar.as_doubles([-3, 2**40], ar.INT), [-3.0, 2.0**40])
