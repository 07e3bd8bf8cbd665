"""Reference for the aggregating additional collectors (reference TermsCollectorManager.fillBucketResultByCount :430-480,
MaxCollectorManager.java:38,117-121, MinCollectorManager.java, SumCollectorManager.java), the checker of
nrtgpu_search_bool_aggs. TEST INFRASTRUCTURE ONLY.

Its inputs are the values of the matching docs that have one: the match set comes from oracle.match_bitmap (every
matching live doc), the values from the column in its stored sortable-long domain, decoded by numpy views:
  - terms: np.unique counts; the `size` buckets with the largest (order_desc) or smallest counts, ties to the smaller
    stored value; total_buckets and other_counts (the docs in buckets not returned). Keys are stored values.
  - max / min: the collectors' loop `if (value > maxValue) maxValue = value` started from UNSET = -Double.MAX_VALUE
    (`value < minValue` from Double.MAX_VALUE), vectorised: NaN and the infinity on the unset side never win.
  - sum: for finite values math.fsum, with the bound n * 2^-53 * sum|v| that any summation order stays within;
    for non-finite values the IEEE result (NaN with a NaN or both infinities, else the infinity)."""
import math

import numpy as np

DBL_MAX = float(np.finfo(np.float64).max)
INT, FLOAT, DOUBLE = 0, 1, 2   # value_type of nrtgpu_aggregation


def decode_float(stored):
    """NumericUtils.sortableIntToFloat of int32-range stored values -> float64"""
    b = np.asarray(stored, np.int64).astype(np.int32)
    b = b ^ ((b >> 31) & np.int32(0x7fffffff))
    return b.view(np.float32).astype(np.float64)


def decode_double(stored):
    """NumericUtils.sortableLongToDouble"""
    b = np.asarray(stored, np.int64)
    b = b ^ ((b >> 63) & np.int64(0x7fffffffffffffff))
    return b.view(np.float64)


def as_doubles(stored, value_type):
    """the doubles the Min / Max / Sum collectors see for stored values of a column of this value type"""
    if value_type == FLOAT:
        return decode_float(stored)
    if value_type == DOUBLE:
        return decode_double(stored)
    return np.asarray(stored, np.int64).astype(np.float64)


def matched_values(column, has, match):
    """stored values of the matching docs that have a value (match: bool [n_docs])"""
    sel = match if has is None else match & (np.asarray(has) != 0)
    return np.asarray(column, np.int64)[sel]


def terms_from_counts(keys, counts, size, order_desc=True):
    """terms result from the per-value counts (keys: stored values, ascending or not; zero counts are empty buckets)"""
    keys, counts = np.asarray(keys, np.int64), np.asarray(counts, np.int64)
    nz = counts > 0
    keys, counts = keys[nz], counts[nz]
    order = np.lexsort((keys, -counts if order_desc else counts))[:size]
    n = len(order)
    out_keys, out_counts = np.zeros(size, np.int64), np.zeros(size, np.int32)
    out_keys[:n], out_counts[:n] = keys[order], counts[order]
    return {"keys": out_keys, "counts": out_counts, "n": n, "total_buckets": len(keys),
            "other_counts": int(counts.sum() - counts[order].sum())}


def terms(values, size, order_desc=True):
    """terms aggregation over the stored values of the collected docs"""
    keys, counts = np.unique(np.asarray(values, np.int64), return_counts=True)
    return terms_from_counts(keys, counts, size, order_desc)


def max_value(v):
    v = np.asarray(v, np.float64)
    v = v[v > -DBL_MAX]
    return float(v.max()) if len(v) else -DBL_MAX


def min_value(v):
    v = np.asarray(v, np.float64)
    v = v[v < DBL_MAX]
    return float(v.min()) if len(v) else DBL_MAX


def sum_value(v):
    """(expected, bound): a sum in any order lies within bound of expected. expected is None when the order decides
    (a partial sum of the finite values may overflow: the reference's single thread is one such order)."""
    v = np.asarray(v, np.float64)
    if np.isnan(v).any() or (np.isposinf(v).any() and np.isneginf(v).any()):
        return math.nan, 0.0
    fin = v[np.isfinite(v)]
    try:
        total, abs_total = math.fsum(fin), math.fsum(np.abs(fin))
    except OverflowError:
        return None, math.inf
    if np.isinf(v).any():
        return float(v[np.isinf(v)][0]), 0.0
    return total, len(v) * 2.0**-53 * abs_total


def sum_ok(got, values):
    """whether `got` is a sum of `values` in some order"""
    expected, bound = sum_value(values)
    if expected is None:   # an overflow gives an infinity, which meets the opposite one (if any) as NaN
        inf = np.asarray(values, np.float64)[np.isinf(values)]
        return (math.isnan(got) or got == inf[0]) if len(inf) else not math.isnan(got)
    if math.isnan(expected) or math.isinf(expected):
        return got == expected or (math.isnan(expected) and math.isnan(got))
    return abs(got - expected) <= bound
