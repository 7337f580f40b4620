"""Differential test of the host planning layer (pinot_b200/csrc/host/pb_host.cpp: PredicateEvaluatorProvider, FilterOperatorUtils,
FilterPlanNode, SortedIndexBasedFilterOperator) against the oracle, on CPU.

The lowered pb_filter_node program of a query (pbh_dump_lowered: exactly what pbh_execute hands to the device) is evaluated by a
few lines of numpy over the decoded columns, and the resulting docId set must equal the oracle's DocIdSetOperator output
(orc_filter_doc_ids) — two independent restatements of the reference's predicate lowering (C++ vs C) meeting in the middle.
"""
import numpy as np
import pytest

from oracle import oracle
from pinot_b200 import datagen, native
from pinot_b200.query import parse_sql
from pinot_b200.segment_writer import DataType
from tests.reference import _column_values, _dict_ids, _raw_values, evaluate_sql  # noqa: F401  (shared with other tests)


def evaluate_lowered(seg, lines):
    """numpy interpreter of the postfix program printed by pbh_dump_lowered; an empty program matches all."""
    n = seg.num_docs
    if not lines:
        return np.ones(n, bool)
    stack = []
    for line in lines:
        op, _, rest = line.partition(" ")
        kv = dict(p.split("=", 1) for p in rest.split()) if rest else {}
        if op == "AND" or op == "OR":
            k = int(kv["n"])
            args, stack = stack[-k:], stack[:-k]
            stack.append(np.logical_and.reduce(args) if op == "AND" else np.logical_or.reduce(args))
        elif op == "NOT":
            stack.append(~stack.pop())
        elif op == "MATCH_ALL":
            stack.append(np.ones(n, bool))
        elif op == "EMPTY":
            stack.append(np.zeros(n, bool))
        elif op == "SCAN_DICT_RANGE":
            ids = _dict_ids(seg.columns[kv["col"]])
            stack.append((ids >= int(kv["lo"])) & (ids < int(kv["hi"])))
        elif op in ("SCAN_DICT_SET", "INVERTED"):
            ids = _dict_ids(seg.columns[kv["col"]])
            member = np.isin(ids, np.array([int(x) for x in kv["ids"].split(",") if x], dtype=np.int64))
            stack.append(~member if kv["excl"] == "1" else member)
        elif op == "SCAN_RAW_RANGE":
            c = seg.columns[kv["col"]]
            v = _raw_values(c)
            if c.data_type in (DataType.INT, DataType.LONG):
                stack.append((v >= int(kv["ilo"])) & (v <= int(kv["ihi"])))
            else:
                v = v.astype(np.float64)
                lo, hi = float(kv["dlo"]), float(kv["dhi"])
                stack.append((v >= lo if kv["dlo_incl"] == "1" else v > lo) & (v <= hi if kv["dhi_incl"] == "1" else v < hi))
        elif op == "SCAN_RAW_SET":
            c = seg.columns[kv["col"]]
            v = _raw_values(c)
            vals = [int(x) for x in kv["vals"].split(",") if x]
            if c.data_type in (DataType.FLOAT, DataType.DOUBLE):      # doubles travel as IEEE-754 bits
                member = np.isin(v.astype(np.float64).view(np.int64), np.array(vals, dtype=np.int64))
            else:
                member = np.isin(v.astype(np.int64), np.array(vals, dtype=np.int64))
            stack.append(~member if kv["excl"] == "1" else member)
        elif op == "SORTED":
            m = np.zeros(n, bool)
            for r in kv["ranges"].split(","):
                if r:
                    s, e = r.split("-")
                    m[int(s):int(e) + 1] = True
            stack.append(m)
        else:
            raise AssertionError(f"unknown node {line!r}")
    assert len(stack) == 1
    return stack[0]


@pytest.fixture(scope="module")
def fuzz_segment():
    seg = datagen.make_segment_synth(7, 30_011, columns=["c1", "c3", "c5", "d0", "s0", "t0", "m0", "x0", "k0"])
    g = native.SegmentGroup([native.StagedSegment(seg)])
    yield seg, g
    g.release()


def _literal(rng, seg, col):
    """a literal for `col`: mostly a value that exists, sometimes one between / outside the dictionary or the value range"""
    c = seg.columns[col]
    if c.has_dictionary:
        d = c.dictionary_values()
        v = d[rng.integers(0, len(d))]
        if c.data_type == DataType.STRING:
            s = v.decode()
            r = rng.random()
            return "'" + (s if r < 0.6 else (s[:2] if r < 0.8 else s + "x")) + "'"
        v = int(v) + int(rng.choice([0, 0, 0, 1, -1, 10**9, -10**9]))
        return str(v)
    if c.data_type in (DataType.DOUBLE, DataType.FLOAT):
        return repr(float(rng.choice([rng.random(), rng.random(), -0.5, 1.5, 0.0])))
    vals = _raw_values(c)
    return str(int(vals[rng.integers(0, len(vals))]) + int(rng.choice([0, 0, 1, -1])))


def _predicate(rng, seg, cols):
    col = str(rng.choice(cols))
    kind = rng.choice(["eq", "neq", "in", "notin", "lt", "le", "gt", "ge", "between"])
    lit = lambda: _literal(rng, seg, col)
    if kind == "eq":
        return f"{col} = {lit()}"
    if kind == "neq":
        return f"{col} <> {lit()}"
    if kind in ("in", "notin"):
        vals = ", ".join(lit() for _ in range(int(rng.integers(1, 6))))
        return f"{col} {'NOT IN' if kind == 'notin' else 'IN'} ({vals})"
    if kind == "between":
        a, b = lit(), lit()
        return f"{col} BETWEEN {a} AND {b}"
    return f"{col} {dict(lt='<', le='<=', gt='>', ge='>=')[kind]} {lit()}"


def _expr(rng, seg, cols, depth):
    if depth == 0 or rng.random() < 0.35:
        p = _predicate(rng, seg, cols)
        return f"NOT {p}" if rng.random() < 0.15 and " IN " not in p and "BETWEEN" not in p else p
    k = int(rng.integers(2, 4))
    op = " AND " if rng.random() < 0.5 else " OR "
    return "(" + op.join(_expr(rng, seg, cols, depth - 1) for _ in range(k)) + ")"


@pytest.mark.parametrize("seed", range(100))
def test_lowered_program_matches_oracle(fuzz_segment, seed):
    seg, g = fuzz_segment
    rng = np.random.default_rng(1000 + seed)
    cols = ["c1", "c3", "c5", "d0", "s0", "t0", "m0", "x0", "k0"]
    for _ in range(6):
        where = _expr(rng, seg, cols, depth=2)
        opts = "SET skipIndexes='c3=inverted'; " if rng.random() < 0.3 else ""
        q = parse_sql(f"{opts}SELECT COUNT(*) FROM t WHERE {where}")
        docs, _ = oracle.filter_doc_ids(seg, q)
        got = np.nonzero(evaluate_lowered(seg, native.dump_lowered(g, q)))[0]
        assert got.tolist() == docs.tolist(), where
        assert np.nonzero(evaluate_sql(seg, q.filter))[0].tolist() == docs.tolist(), where      # ... and both equal the SQL semantics


# ---- enableNullHandling: three restatements of the operators' three-valued doc sets ----

def _null_mask(seg, col):
    v = getattr(seg.columns[col], "null_value_vector", None)
    m = np.zeros(seg.num_docs, bool)
    if v is not None:
        out = np.zeros(seg.num_docs, dtype=np.uint32)
        n = oracle.lib().orc_roaring_to_doc_ids(v.ctypes.data, v.size, out.ctypes.data, out.size)
        m[out[:n]] = True
    return m


def evaluate_lowered_nh(seg, lines):
    """evaluate_lowered plus the BITMAP leaves of null-value vectors"""
    plain, patched = [], {}
    for i, line in enumerate(lines):
        if line.startswith("BITMAP "):
            kv = dict(p.split("=", 1) for p in line.split()[1:3])
            m = _null_mask(seg, kv["col"])
            patched[i] = ~m if kv["excl"] == "1" else m
    # run the stock interpreter with the bitmap leaves swapped for a marker it understands
    n = seg.num_docs
    stack = []
    for i, line in enumerate(lines):
        if i in patched:
            stack.append(patched[i])
            continue
        op = line.split(" ", 1)[0]
        if op in ("AND", "OR"):
            k = int(line.split("n=")[1])
            args, stack = stack[-k:], stack[:-k]
            stack.append(np.logical_and.reduce(args) if op == "AND" else np.logical_or.reduce(args))
        elif op == "NOT":
            stack.append(~stack.pop())
        else:
            stack.append(evaluate_lowered(seg, [line]))
    if not lines:
        return np.ones(n, bool)
    assert len(stack) == 1
    return stack[0]


def operator_model(seg, node):
    """(trues, nulls, falses) of a filter node as the reference's operators define them: BaseFilterOperator.java:88-113,
    BaseColumnFilterOperator.java:46-70, And / Or / NotFilterOperator, FilterOperatorUtils.java:74-88 -- in numpy over the
    decoded values."""
    from pinot_b200.query import And, Not, Or, PredicateType
    n = seg.num_docs
    zero = np.zeros(n, bool)
    if isinstance(node, Not):
        t, _, f = operator_model(seg, node.child)
        return f, zero, t
    if isinstance(node, (And, Or)):
        kids = [operator_model(seg, c) for c in node.children]
        if isinstance(node, And):
            t = np.logical_and.reduce([k[0] for k in kids])
            f = ~np.logical_and.reduce([k[0] | k[1] for k in kids])
        else:
            t = np.logical_or.reduce([k[0] for k in kids])
            f = ~np.logical_or.reduce([k[0] | k[1] for k in kids])
        return t, zero, f                                   # (And / Or do not override getNulls())
    nulls = _null_mask(seg, node.column)
    if node.type in (PredicateType.IS_NULL, PredicateType.IS_NOT_NULL):
        t = nulls if node.type == PredicateType.IS_NULL else ~nulls
        return t, zero, ~t
    base = evaluate_sql(seg, node)                          # two-valued, on the stored values (default null values included)
    c = seg.columns[node.column]
    if not c.has_dictionary and node.type == PredicateType.RANGE and c.data_type in (DataType.INT, DataType.LONG):
        # the raw integral range evaluator folds its bounds to inclusive ones and is alwaysFalse when they cross
        # (RangePredicateEvaluatorFactory.java:331-366): an EmptyFilterOperator, which has no nulls
        lo = None if node.lower is None else int(node.lower) + (0 if node.lower_inclusive else 1)
        hi = None if node.upper is None else int(node.upper) - (0 if node.upper_inclusive else 1)
        if lo is not None and hi is not None and lo > hi:
            return zero, zero, ~zero
    if c.has_dictionary and not base.any():                 # alwaysFalse: EmptyFilterOperator
        return zero, zero, ~zero
    if c.has_dictionary and base.all():                     # alwaysTrue: the flipped null bitmap (or MatchAll), no nulls of its own
        t = ~nulls
        return t, zero, ~t
    t = base & ~nulls
    return t, nulls, ~(t | nulls)


@pytest.fixture(scope="module")
def nullable_fuzz_segment():
    from pinot_b200.segment_writer import build_column, make_segment, with_nulls
    rng = np.random.default_rng(77)
    n = 9_001
    int_null = np.iinfo(np.int32).min
    def nullable(name, dt, values, p, default, **kw):
        nl = rng.random(n) < p
        return with_nulls(build_column(name, dt, np.where(nl, default, values), **kw), nl)
    s_vals = np.sort(rng.integers(0, 30, n)).astype(np.int32)
    s_null = np.zeros(n, bool); s_null[:40] = True                                      # the nulls of the sorted column carry its smallest value
    cols = [nullable("a", DataType.INT, rng.integers(-4, 5, n).astype(np.int32), 0.25, int_null),
            nullable("b", DataType.INT, rng.integers(0, 12, n).astype(np.int32), 0.15, int_null, inverted=True),
            nullable("r", DataType.LONG, rng.integers(-20, 20, n).astype(np.int64), 0.2, 0, dictionary=False),
            nullable("x", DataType.DOUBLE, np.round(rng.normal(0, 2, n), 1), 0.3, 0.0, dictionary=False),
            with_nulls(build_column("s", DataType.INT, np.where(s_null, s_vals.min(), s_vals).astype(np.int32)), s_null),
            build_column("d", DataType.INT, rng.integers(0, 5, n).astype(np.int32))]
    seg = make_segment("nhfuzz", cols)
    g = native.SegmentGroup([native.StagedSegment(seg)])
    yield seg, g
    g.release()


def _expr_nh(rng, seg, cols, depth):
    r = rng.random()
    if depth == 0 or r < 0.3:
        col = str(rng.choice(cols))
        if rng.random() < 0.2:
            return f"{col} IS {'NOT ' if rng.random() < 0.5 else ''}NULL"
        return _predicate(rng, seg, [col])
    if r < 0.5:
        return "NOT (" + _expr_nh(rng, seg, cols, depth - 1) + ")"
    k = int(rng.integers(2, 4))
    op = " AND " if rng.random() < 0.5 else " OR "
    return "(" + op.join(_expr_nh(rng, seg, cols, depth - 1) for _ in range(k)) + ")"


@pytest.mark.parametrize("seed", range(60))
def test_null_handling_lowering_matches_oracle_and_operator_model(nullable_fuzz_segment, seed):
    """enableNullHandling: the trues program of the host layer (C++), the oracle's operator tree (C) and a numpy model of the
    operators' getTrues / getNulls / getFalses must select the same docs -- on trees with NOT at any depth, IS [NOT] NULL
    leaves, sorted / inverted / raw / plain dictionary columns, always-true and always-false predicates."""
    seg, g = nullable_fuzz_segment
    rng = np.random.default_rng(5000 + seed)
    cols = ["a", "b", "r", "x", "s", "d"]
    for _ in range(6):
        where = _expr_nh(rng, seg, cols, depth=3)
        q = parse_sql(f"SET enableNullHandling=true; SELECT COUNT(*) FROM t WHERE {where}")
        docs, _ = oracle.filter_doc_ids(seg, q)
        got = np.nonzero(evaluate_lowered_nh(seg, native.dump_lowered(g, q)))[0]
        assert got.tolist() == docs.tolist(), where
        assert np.nonzero(operator_model(seg, q.filter)[0])[0].tolist() == docs.tolist(), where


def test_edge_literals_on_dictionary_columns():
    """Literals at the edges of the types, on dictionaries that hold both zeros, infinities, denormals and the extremes of
    long: the host layer (C++) and the oracle (C) must lower them to the same docs, and to what the reference's dictionaries
    do -- Float.parseFloat rounds the literal before the search (FloatDictionary.java:43-45: "0.1" finds 0.1f), comparisons are
    numeric (0.0 finds the first zero the binary search meets), a long that does not parse fails the query."""
    from pinot_b200.segment_writer import build_dict_column, make_segment
    rng = np.random.default_rng(0)
    n = 5000
    xv = np.array([-np.inf, -1e308, -1.5, -0.0, 0.0, 1e-320, 2.5, 1e308, np.inf])
    kv = np.array([np.iinfo(np.int64).min, -5, 0, 7, np.iinfo(np.int64).max], dtype=np.int64)
    fv = np.array([-3.25, -0.0, 0.0, 0.1, 16777216.0, 16777218.0], dtype=np.float32)
    xi, ki, fi = (rng.integers(0, len(v), n).astype(np.uint32) for v in (xv, kv, fv))
    seg = make_segment("edge", [build_dict_column("x", DataType.DOUBLE, xv, xi), build_dict_column("k", DataType.LONG, kv, ki),
                                build_dict_column("f", DataType.FLOAT, fv, fi)])
    g = native.SegmentGroup([native.StagedSegment(seg)])
    x, k, f = xv[xi], kv[ki], fv[fi]
    F = np.float32
    cases = {
        "x > -0.0": x > 0, "x <= -0.0": x <= 0,
        "x > 1e308": x > 1e308, "x >= 1e309": np.isinf(x) & (x > 0), "x < -1e309": np.zeros(n, bool), "x = 1e-320": x == 1e-320,
        "x > 1e-321": x > 1e-321, "x NOT IN (2.5, 1e308)": ~np.isin(x, [2.5, 1e308]),
        "k = -9223372036854775808": k == np.iinfo(np.int64).min, "k <= 9223372036854775807": np.ones(n, bool),
        "k > 9223372036854775806": k == np.iinfo(np.int64).max, "k BETWEEN -5 AND 7": (k >= -5) & (k <= 7),
        "k IN (0, 9223372036854775807)": np.isin(k, [0, np.iinfo(np.int64).max]), "k > 6": k > 6,
        "f = 0.1": f == F(0.1), "f > 0.1": f > F(0.1), "f >= 0.1": f >= F(0.1), "f < 0.1": f < F(0.1),
        "f = 16777217": f == F(16777217), "f > 16777217": f > F(16777217), "f BETWEEN 16777216 AND 16777217": (f >= F(16777216)) & (f <= F(16777217)),
        "f <> 0.1": f != F(0.1), "f = 0.10000000149011612": f == F(0.1),
    }
    for where, exp in cases.items():
        q = parse_sql("SELECT COUNT(*) FROM t WHERE " + where)
        docs, _ = oracle.filter_doc_ids(seg, q)
        got = np.nonzero(evaluate_lowered(seg, native.dump_lowered(g, q)))[0]
        assert got.tolist() == docs.tolist() == np.nonzero(exp)[0].tolist(), where
    # equality with a zero: whichever zero the reference's binary search meets first -- the two restatements must agree
    # (the same for a range that starts or ends AT a zero: the found entry is the boundary, the other zero falls on one side)
    for where in ("x = 0.0", "x = -0.0", "x <> 0.0", "x IN (0.0)", "x IN (-0.0, 2.5)", "f IN (0.1, -0.0)", "f <> 0.0",
                  "x >= 0.0", "x < 0.0", "x BETWEEN -0.0 AND 0.0"):
        q = parse_sql("SELECT COUNT(*) FROM t WHERE " + where)
        assert np.nonzero(evaluate_lowered(seg, native.dump_lowered(g, q)))[0].tolist() == oracle.filter_doc_ids(seg, q)[0].tolist(), where
    # Long.parseLong("9223372036854775808") throws in the reference: the plan maker declines, the oracle refuses
    q = parse_sql("SELECT COUNT(*) FROM t WHERE k = 9223372036854775808")
    assert not native.is_eligible(g, q)
    with pytest.raises(ValueError):
        oracle.filter_doc_ids(seg, q)
    g.release()


def test_edge_literals_on_raw_columns():
    """The same on raw (no-dictionary) INT / LONG / FLOAT / DOUBLE columns holding the extremes, both zeros, infinities, NaN
    and the smallest denormal: integral ranges are folded to inclusive bounds (RangePredicateEvaluatorFactory.java:331-366),
    FLOAT bounds are Float.parseFloat(bound), NaN matches no range and no equality."""
    from pinot_b200.segment_writer import build_column, make_segment
    rng = np.random.default_rng(1)
    n = 4000
    i = rng.choice(np.array([np.iinfo(np.int32).min, -7, 0, 5, np.iinfo(np.int32).max], dtype=np.int32), n)
    l = rng.choice(np.array([np.iinfo(np.int64).min, -7, 0, 5, np.iinfo(np.int64).max], dtype=np.int64), n)
    f = rng.choice(np.array([-np.inf, -0.0, 0.0, 0.1, 16777216.0, 3.4e38, np.inf, np.nan], dtype=np.float32), n)
    d = rng.choice(np.array([-np.inf, -0.0, 0.0, 0.1, 1e308, np.inf, np.nan, 5e-324]), n)
    seg = make_segment("rawedge", [build_column("i", DataType.INT, i, dictionary=False), build_column("l", DataType.LONG, l, dictionary=False),
                                   build_column("f", DataType.FLOAT, f, dictionary=False), build_column("d", DataType.DOUBLE, d, dictionary=False)])
    g = native.SegmentGroup([native.StagedSegment(seg)])
    F = np.float32
    imax, imin, lmax, lmin = np.iinfo(np.int32).max, np.iinfo(np.int32).min, np.iinfo(np.int64).max, np.iinfo(np.int64).min
    with np.errstate(invalid="ignore"):
        cases = {
            "i > 2147483646": i == imax, "i >= 2147483647": i == imax, "i > 2147483647": np.zeros(n, bool), "i < -2147483648": np.zeros(n, bool),
            "i <= -2147483648": i == imin, "i = 2147483647": i == imax, "i <> -2147483648": i != imin, "i IN (5, 2147483647)": np.isin(i, [5, imax]),
            "i BETWEEN 5 AND 4": np.zeros(n, bool), "i > -8 AND i < 6": (i > -8) & (i < 6),
            "l > 9223372036854775806": l == lmax, "l > 9223372036854775807": np.zeros(n, bool), "l < -9223372036854775808": np.zeros(n, bool),
            "l = -9223372036854775808": l == lmin, "l NOT IN (0, 5)": ~np.isin(l, [0, 5]),
            "f > 0.1": f > F(0.1), "f >= 0.1": f >= F(0.1), "f = 0.1": f == F(0.1), "f < 0.1": f < F(0.1), "f <> 0.1": f != F(0.1),
            "f > 3.4e38": f > F(3.4e38), "f >= 3.5e38": f >= F(np.inf), "f = 16777217": f == F(16777217), "f > -0.0": f > 0, "f >= 0.0": f >= 0,
            "f < 0.0": f < 0, "f <= -0.0": f <= 0, "f BETWEEN 0 AND 0.1": (f >= 0) & (f <= F(0.1)),
            "d > 0.1": d > 0.1, "d = 0.1": d == 0.1, "d >= 1e308": d >= 1e308, "d > 1e308": d > 1e308, "d < 5e-324": d < 5e-324,
            "d <= 5e-324": d <= 5e-324, "d = 5e-324": d == 5e-324, "d > -0.0": d > 0, "d >= 0.0": d >= 0, "d < 0.0": d < 0, "d <= -0.0": d <= 0,
            "d <> 0.1": d != 0.1, "d BETWEEN -1 AND 1": (d >= -1) & (d <= 1),
            "d = 0.0": d == 0, "d <> -0.0": d != 0, "f = -0.0": f == 0,                                      # == : both zeros
            "d IN (0.0, 0.1)": np.isin(d.view(np.int64), np.array([0.0, 0.1]).view(np.int64)),                   # DoubleSet: by bit pattern
            "d NOT IN (0.1, 1e308)": ~np.isin(d.view(np.int64), np.array([0.1, 1e308]).view(np.int64)),
        }
    for where, exp in cases.items():
        q = parse_sql("SELECT COUNT(*) FROM t WHERE " + where)
        docs, _ = oracle.filter_doc_ids(seg, q)
        got = np.nonzero(evaluate_lowered(seg, native.dump_lowered(g, q)))[0]
        assert got.tolist() == docs.tolist() == np.nonzero(exp)[0].tolist(), where
    g.release()


@pytest.mark.parametrize("seed", range(20))
def test_null_handling_clause_programs(nullable_fuzz_segment, seed):
    """enableNullHandling, aggregation side: every aggregation over a nullable column runs under the clause "its own FILTER
    clause (trues) AND <column> IS NOT NULL"; functions with the same pair share a clause.  The lowered clause programs against
    the numpy model of the operators."""
    seg, g = nullable_fuzz_segment
    rng = np.random.default_rng(9000 + seed)
    cols = ["a", "b", "r", "x", "s", "d"]
    aggs = []
    for _ in range(int(rng.integers(2, 6))):
        fn = str(rng.choice(["SUM", "MIN", "MAX", "AVG", "COUNT"]))
        col = str(rng.choice(["a", "r", "x", "d", "*"] if fn == "COUNT" else ["a", "r", "x", "d"]))
        flt = f" FILTER(WHERE {_expr_nh(rng, seg, cols, depth=2)})" if rng.random() < 0.5 else ""
        aggs.append(f"{fn}({col}){flt}")
    q = parse_sql(f"SET enableNullHandling=true; SELECT {', '.join(aggs)} FROM t WHERE d >= 0")
    n_clauses, clause_of = native.clause_plan(g, q)
    seen = {}
    for a, agg in enumerate(q.aggregations):
        nullable = agg.column is not None and getattr(seg.columns[agg.column], "null_value_vector", None) is not None
        if agg.filter is None and not nullable:
            assert clause_of[a] == -1, aggs[a]
            continue
        k = clause_of[a]
        assert 0 <= k < n_clauses, aggs[a]
        exp = operator_model(seg, agg.filter)[0] if agg.filter is not None else np.ones(seg.num_docs, bool)
        if nullable:
            exp = exp & ~_null_mask(seg, agg.column)
        got = evaluate_lowered_nh(seg, native.dump_lowered(g, q, k))
        assert np.array_equal(got, exp), aggs[a]
        key = (repr(agg.filter), agg.column if nullable else None)
        assert seen.setdefault(key, k) == k, "functions with the same (clause, column) pair share a clause"
    assert n_clauses == len(set(seen.values()))
