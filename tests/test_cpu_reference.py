"""tests/reference.py (the exact reference the device fuzz is held to) against the oracle, on the fuzz tables and queries of
tests/test_gpu_fuzz.py with the same seeds -- so the reference is validated on a machine without a GPU.  CPU only.

The one divergence allowed: a keyless MIN / MAX over inputs that hold a NaN, where the oracle folds with Math.min / Math.max
(the result is NaN) and the reference keeps the group-by semantics the device documents for keyless aggregation too."""
import math

import numpy as np
import pytest

from oracle import oracle
from pinot_b200.query import AggOp, parse_sql
from tests import fuzz_gen
from tests.parity import combined_rows, oracle_rows
from tests.reference import SumRef, assert_matches_reference, check_sum, concat, keyless_nan_minmax, reference, without_aggregations

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
