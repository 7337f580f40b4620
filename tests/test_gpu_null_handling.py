"""enableNullHandling on the device: the host layer folds the three-valued filter into its trues program and gives every
aggregation over a nullable column the implicit clause "<column> IS NOT NULL"; the device keeps the inputs every function saw
(0 = SQL NULL).  Compared with the oracle (itself pinned to the reference's fixtures in tests/test_cpu_null_handling.py) and with
those fixtures directly."""
import numpy as np
import pytest

from pinot_b200 import native
from pinot_b200.query import parse_sql
from pinot_b200.segment_writer import DataType, build_column, make_segment, with_nulls
from tests.parity import check_query
from tests.test_cpu_null_handling import INT_NULL, NH, one_column_fixture, records_fixture, two_column_fixture

pytestmark = pytest.mark.gpu


def _count(seg, where, nh=True):
    native.init()
    g = native.SegmentGroup([native.StagedSegment(seg)])
    res = native.execute(g, parse_sql((NH if nh else "") + f"SELECT COUNT(*) FROM t WHERE {where}"), 0)
    n = res.tables[0].rows()[()][0]
    res.free()
    return n


def test_reference_filter_fixtures_on_the_device():
    seg, _ = two_column_fixture()
    assert _count(seg, "c1 > 0 OR c2 < 0") == 3                      # NullHandlingEnabledQueriesTest.testOrFiltering
    assert _count(seg, "NOT (c1 > 0 AND c2 < 0)") == 3               # testNotAndFiltering
    assert _count(seg, "NOT (c1 > 0 OR c2 < 0)") == 1                # testNotOrFiltering
    assert _count(one_column_fixture([None, -1, 1]), "NOT (c1 = 1)") == 1                      # testNotFiltering
    assert _count(one_column_fixture([-1, None], sort=True), "c1 < 0") == 1                    # testRangeFiltering
    assert _count(one_column_fixture([None, INT_NULL], sort=True), f"c1 = {INT_NULL}") == 1    # testEqualFiltering
    assert _count(seg, "NOT (c1 > 0 OR c2 < 0)", nh=False) == 2


@pytest.mark.parametrize("dtype,base", [(DataType.INT, 7), (DataType.DOUBLE, 0.6180339887)])
def test_reference_aggregation_expectations_on_the_device(dtype, base):
    native.init()
    seg, v, keys, nulls = records_fixture(base, dtype, True)
    segs = [seg]
    exact = dtype == DataType.INT                  # (sums of doubles: the device adds in another order)
    check_query(segs, NH + "SELECT COUNT(column), MIN(column), MAX(column), AVG(column), SUM(column) FROM t", exact_float=exact)
    check_query(segs, NH + "SELECT key, SUM(column), MIN(column), MAX(column), COUNT(column) FROM t GROUP BY key LIMIT 10", exact_float=exact)
    g = native.SegmentGroup([native.StagedSegment(seg)])
    r = native.execute(g, parse_sql(NH + "SELECT key, SUM(column), MIN(column), MAX(column), COUNT(column) FROM t GROUP BY key LIMIT 10"), 0)
    rows = r.tables[0].rows()
    assert rows[(0,)] == [None, None, None, 0]                       # the all-null group: SUM / MIN / MAX are SQL NULL, COUNT(col) = 0
    assert rows[(1,)][3] == 250 and rows[(2,)][3] == 250             # NullEnabledQueriesTest :281-330
    r.free()


FUZZ_QUERIES = [
    "SELECT d, COUNT(*), COUNT(a), SUM(a), MIN(b), MAX(x), AVG(x) FROM t WHERE NOT (a > 2) GROUP BY d LIMIT 100",
    "SELECT d, SUM(b), AVG(a), DISTINCTCOUNT(a) FROM t WHERE NOT (a IN (1, 2, 3) OR x < 0.5) AND s > 3 GROUP BY d LIMIT 100",
    "SELECT COUNT(*), SUM(x), MIN(a), MAX(b), COUNT(b) FROM t WHERE a IS NULL OR NOT (b BETWEEN 100 AND 900)",
    "SELECT d, COUNT(*), SUM(b) FILTER(WHERE NOT (a = 0)), MAX(x) FILTER(WHERE b > 500), COUNT(x) FROM t WHERE NOT (x > 4 AND a < 0) GROUP BY d LIMIT 100",
    "SELECT COUNT(*), SUM(a), AVG(b) FROM t WHERE NOT (NOT (a < 0) AND NOT (x IS NULL)) AND s < 35",
    "SELECT d, MIN(x), MAX(a) FROM t WHERE a <> 3 AND NOT (s = 7) GROUP BY d LIMIT 100",
    "SELECT SUM(a), MIN(x), COUNT(a) FROM t WHERE a > 100",                     # nothing matches: every function is NULL, COUNT 0
]


def fuzz_segments():
    """three segments of random nullable columns (dictionary, raw, sorted, inverted), one without any null vector"""
    rng = np.random.default_rng(21)
    segs = []
    for si, n in enumerate((20_011, 9_000, 14_500)):
        d = rng.integers(0, 7, n).astype(np.int32)
        a = rng.integers(-5, 6, n).astype(np.int32)
        b = rng.integers(0, 1000, n).astype(np.int64)
        x = np.round(rng.normal(0, 3, n), 1)
        s = np.sort(rng.integers(0, 40, n)).astype(np.int32)
        an, bn, xn, sn = (rng.random(n) < p for p in (0.2, 0.1, 0.3, 0.05))
        if si == 1:
            an[:] = False; bn[:] = False; xn[:] = False; sn[:] = False          # a segment whose columns have no null-value vector
        sn &= (s == s.min())                                                       # nulls of the sorted column carry its smallest value
        cols = [build_column("d", DataType.INT, d),
                with_nulls(build_column("a", DataType.INT, np.where(an, INT_NULL, a).astype(np.int32), inverted=True), an),
                with_nulls(build_column("b", DataType.LONG, np.where(bn, 0, b), dictionary=False), bn),
                with_nulls(build_column("x", DataType.DOUBLE, np.where(xn, 0.0, x)), xn),
                with_nulls(build_column("s", DataType.INT, s), sn)]
        segs.append(make_segment(f"nh{si}", cols))
    return segs


def test_null_handling_fuzz_against_the_oracle():
    """Random nullable columns (fuzz_segments), random filter trees with NOT / AND / OR / IS NULL, filtered aggregations on
    top, several segments, per segment and combined."""
    native.init()
    segs = fuzz_segments()
    for sql in FUZZ_QUERIES:
        # (a query with FILTER clauses of its own reports plain statistics under null handling, the reference its swim-lanes)
        check_query(segs, NH + sql, exact_float=False, check_stats="FILTER(" not in sql)
    # and the same statements without the option still run two-valued
    check_query(segs, FUZZ_QUERIES[0], exact_float=False)
