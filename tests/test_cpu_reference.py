"""tests/reference.py (the exact reference the device fuzz is held to) against the oracle, on the fuzz tables and queries of
tests/test_gpu_fuzz.py with the same seeds -- so the reference is validated on a machine without a GPU.  CPU only.

The one divergence allowed: a keyless MIN / MAX over inputs that hold a NaN, where the oracle folds with Math.min / Math.max
(the result is NaN) and the reference keeps the group-by semantics the device documents for keyless aggregation too."""
import dataclasses
import math

import numpy as np
import pytest

from oracle import oracle
from pinot_b200.query import AggOp, Aggregation, parse_sql
from pinot_b200.segment_writer import DataType, build_column, make_segment
from tests import fuzz_gen
from tests.parity import combined_rows, oracle_rows
from tests.reference import (Col, SumRef, assert_matches_reference, check_sum, concat, keyless_nan_minmax, limit_reference, order_double,
                             order_interval, reference, trim_bounds, without_aggregations)

SEEDS = range(8)                  # the seeds of tests/test_gpu_fuzz.py
QUERIES_PER_SEED = 6


def _compare(got, ref, q, skip, what):
    """assert_matches_reference without the aggregations in `skip`; those must be NaN in the oracle's row or match"""
    for a in skip:
        for k, row in got.items():
            assert math.isnan(row[a]) or row[a] == ref[k][a], f"{what}: keyless {q.aggregations[a]}: {row[a]!r}"
    assert_matches_reference(*without_aggregations(got, ref, q, skip), what)


@pytest.mark.parametrize("seed", SEEDS)
def test_reference_matches_oracle_on_fuzz_tables(seed):
    segs, srcs, _ = fuzz_gen.make_tables(seed)
    rng = np.random.default_rng(seed)
    for qi in range(QUERIES_PER_SEED):
        sql = fuzz_gen.make_query(rng, srcs[0])
        q = parse_sql(sql)
        orc = [oracle.execute(s, q) for s in segs]
        skip = keyless_nan_minmax(q, srcs)
        for i, (o, src) in enumerate(zip(orc, srcs)):
            _compare(oracle_rows(o), reference(src, q), q, skip, f"seed {seed} query {qi} segment {i}: {sql}")
        _compare(combined_rows(oracle.combine(orc), q), reference(concat(srcs), q), q, skip, f"seed {seed} query {qi} merged: {sql}")


def _key_space(seg, q):
    return int(np.prod([seg.columns[c].cardinality for c in q.group_by], dtype=object))


def _check_limit_against_oracle(seg, src, q, what):
    """a dense per-segment table: the reference's first `limit` keys in doc order and its flag equal the oracle's holder.
    (Without FILTER clauses: Pinot's filtered group-by feeds the key generator lane by lane, so under a reachable limit
    its groups depend on the lanes' order; the device keeps the first keys in doc order, DESIGN.md §4.5.)"""
    aggs = [a for a in q.aggregations if a.filter is None] or [Aggregation(AggOp.COUNT, None)]
    q = dataclasses.replace(q, aggregations=aggs)
    lref = limit_reference(src, q, "dense", _key_space(seg, q))
    o = oracle.execute(seg, q)
    assert lref.exact
    assert_matches_reference(oracle_rows(o), lref.rows, q, what)
    assert o.stats["num_groups_limit_reached"] == int(lref.reached), what
    return lref


@pytest.mark.parametrize("seed", range(4))
def test_limit_reference_matches_oracle_on_fuzz_tables(seed):
    """the shaped queries of tests/test_gpu_result_shaping.py over dictionary keys (their key space is known)"""
    segs, srcs, _ = fuzz_gen.make_tables(seed)
    rng = np.random.default_rng(1_000 + seed)
    checked = 0
    for qi in range(5):
        sql = fuzz_gen.make_shaped_query(rng, srcs[0])
        q = parse_sql(sql)
        if any(not segs[0].columns[c].has_dictionary for c in q.group_by) or _key_space(segs[0], q) > 2 ** 22:
            continue
        for i, (seg, src) in enumerate(zip(segs, srcs)):
            _check_limit_against_oracle(seg, src, q, f"seed {seed} query {qi} segment {i}: {sql}")
        checked += 1
    if seed == 0:
        assert checked


def test_limit_reference_matches_oracle_on_hand_cases():
    """limits 1, groups - 1, groups and key space - 1 over a key whose first docs come in an order unrelated to its
    values, under a filter, with a FILTER clause that leaves some groups nothing"""
    n = 5_000
    r = np.random.default_rng(3)
    k = r.integers(0, 40, n)
    k[:50] = r.permutation(50)                    # 50 dictionary entries
    f = r.integers(0, 4, n)
    v = r.integers(-100, 100, n)
    seg = make_segment("lim", [build_column("k", DataType.INT, k.astype(np.int32)), build_column("f", DataType.INT, f.astype(np.int32)),
                               build_column("v", DataType.INT, v.astype(np.int32))])
    src = {"k": Col(k, DataType.INT), "f": Col(f, DataType.INT), "v": Col(v, DataType.INT)}
    groups = len(np.unique(k[f < 3]))
    for limit in (1, groups - 1, groups, 49, 50):
        q = parse_sql(f"SET numGroupsLimit = {limit}; SELECT k, COUNT(*), SUM(v), AVG(v) FILTER(WHERE k > 45), MIN(v) "
                      f"FROM t WHERE f < 3 GROUP BY k LIMIT 1000")
        lref = _check_limit_against_oracle(seg, src, q, f"limit {limit}")
        assert len(lref.rows) == min(limit, groups) and lref.reached == (groups >= limit)
    # merged dense and hash: every group, the flag once the groups reach the limit
    q = parse_sql("SET numGroupsLimit = 10; SELECT k, COUNT(*) FROM t GROUP BY k LIMIT 1000")
    assert limit_reference(src, q, "merged") == (reference(src, q), True, 50, True)
    h = limit_reference(src, q, "hash")
    assert not h.exact and h.at_most == 10 and h.reached


def test_trim_bounds_on_points_are_the_sorted_cut():
    """trim_bounds against brute-force sorting, on exactly ordered values with many ties, and on intervals against the
    pairwise definition"""
    rng = np.random.default_rng(0)
    for _ in range(500):
        n = int(rng.integers(1, 40))
        v = rng.integers(-4, 5, n)
        size = int(rng.integers(1, n + 3))
        must, never = trim_bounds(v, v, size)
        want = v >= sorted(v, reverse=True)[size - 1] if size <= n else np.ones(n, bool)
        assert (must == want).all() and (never == ~want).all(), (v, size)
        lo = rng.integers(-6, 6, n)
        hi = lo + rng.integers(0, 3, n)
        must, never = trim_bounds(lo, hi, size)
        for g in range(n):
            could = sum(1 for h in range(n) if h != g and hi[h] > lo[g])
            certain = sum(1 for h in range(n) if lo[h] > hi[g])
            assert must[g] == (could < size) and never[g] == (certain >= size)


def test_order_values_follow_double_compare_and_final_results():
    seq = [-math.inf, -1e300, -1.0, -5e-324, -0.0, 0.0, 5e-324, 2.0, math.inf, math.nan]
    assert [order_double(x) for x in seq] == sorted(order_double(x) for x in seq)
    assert len({order_double(x) for x in seq}) == len(seq)
    q = parse_sql("SELECT k, AVG(v) FILTER(WHERE f = 1), MIN(v), SUM(v) FROM t GROUP BY k ORDER BY AVG(v) FILTER(WHERE f = 1) LIMIT 1")
    assert q.order_by == [(1, 0, False)]
    empty = SumRef(0, 0, 0.0, 0.0, True)
    assert order_interval(q, (1,), [empty, 0.0, SumRef(6, 3, 6.0, 2.0, True)]) == (order_double(-math.inf),) * 2
    assert order_interval(q, (1,), [SumRef(-7, 2, 7.0, 4.0, True), 0.0, None]) == (order_double(-3.5),) * 2
    lo, hi = order_interval(q, (1,), [SumRef(0.3, 3, 0.9, 0.5, False), 0.0, None])
    assert lo < order_double(0.1) < hi
    q = parse_sql("SELECT k, MIN(v) FROM t GROUP BY k ORDER BY MIN(v) DESC LIMIT 1")
    assert order_interval(q, (1,), [0.0]) == (order_double(-0.0), order_double(0.0))
    assert order_interval(q, (1,), [math.inf]) == (order_double(math.inf),) * 2
    with pytest.raises(ValueError):
        parse_sql("SELECT k, AVG(v) FILTER(WHERE f = 1) FROM t GROUP BY k ORDER BY AVG(v) FILTER(WHERE f = 2) LIMIT 1")


def test_shaped_queries_trim_only_past_the_small_key_sets():
    _, srcs, _ = fuzz_gen.make_tables(0, max_total=5_000)
    rng = np.random.default_rng(1)
    for _ in range(200):
        q = parse_sql(fuzz_gen.make_shaped_query(rng, srcs[0]))
        assert q.order_by and 1 <= q.limit <= 4
        for combined in (False, True):
            size, thr = q.trim(combined)
            assert 6 <= size <= 20 and thr <= 80, (size, thr)


def test_keyless_min_max_over_nan_is_the_one_divergence():
    segs, srcs, _ = fuzz_gen.make_tables(0, max_total=5_000)
    q = parse_sql("SELECT MIN(edbl), MAX(edbl), MIN(enan), MAX(enan) FROM t")
    o = oracle_rows(oracle.execute(segs[0], q))[()]
    r = reference(srcs[0], q)[()]
    assert all(math.isnan(x) for x in o)
    assert r == [-math.inf, math.inf, math.inf, -math.inf]


def test_sum_rules():
    """check_sum: exact for small integers, the order-independent bound otherwise, NaN / infinity rules"""
    assert check_sum(6.0, SumRef(6, 3, 6.0, 3.0, True)) is None
    assert check_sum(6.0000000000000009, SumRef(6, 3, 6.0, 3.0, True)) is not None           # integers: exact
    big = 2 ** 52 + 1                                                                           # n * max|x| >= 2^53: bound
    assert check_sum(float(3 * big), SumRef(3 * big, 3, 3.0 * big, float(big), True)) is None
    x = [1e16, 1.0, -1e16]                                                                     # cancellation
    r = SumRef(math.fsum(x), 3, sum(abs(v) for v in x), 1e16, False)
    assert check_sum(0.0, r) is None and check_sum(1.0, r) is None and check_sum(8.0, r) is not None
    assert check_sum(math.nan, SumRef(math.nan, 2, 0.0, 0.0, False)) is None
    assert check_sum(math.inf, SumRef(math.nan, 2, 0.0, 0.0, False)) is not None
    assert check_sum(-math.inf, SumRef(-math.inf, 2, 1.0, 1.0, False)) is None
    assert check_sum(math.inf, SumRef(-math.inf, 2, 1.0, 1.0, False)) is not None
    # a dropped doc in a 10^6-term sum: within 1e-6 relative, far outside the bound
    n, s = 10 ** 6, 0.5 * 10 ** 6
    assert check_sum(s - 0.5, SumRef(s, n, s, 1.0, False)) is not None
