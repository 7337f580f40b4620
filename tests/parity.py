"""Helpers that compare the CUDA path (through the C ABI) with the oracle on the same segments."""
from typing import Dict, List, Sequence

import numpy as np

from oracle import oracle
from pinot_b200 import native
from pinot_b200.query import AggOp, And, Not, Or, PredicateType, QueryContext, parse_sql
from tests import reference

REL_TOL = 1e-6   # BASELINE.json north_star: double SUM/AVG within 1e-6 relative; everything integral bit-exact


def oracle_rows(r: "oracle.OracleResult") -> Dict[tuple, list]:
    """key -> per-aggregation value in the same shape as native.ResultTable.rows()."""
    q = r.query
    keys = r.decoded_keys() if q.group_by else [()]
    nh = getattr(q, "null_handling", False)      # longs then hold the inputs every function saw: 0 = SQL NULL
    out = {}
    for g, k in enumerate(keys):
        row = []
        for a, agg in enumerate(q.aggregations):
            if agg.op in (AggOp.COUNT, AggOp.DISTINCTCOUNT):
                row.append(int(r.longs[a][g]))
            elif nh and int(r.longs[a][g]) == 0:
                row.append(None)
            elif agg.op == AggOp.AVG:
                row.append((float(r.doubles[a][g]), int(r.longs[a][g])))
            else:
                row.append(float(r.doubles[a][g]))
        out[k] = row
    return out


def combined_rows(table: Dict[tuple, list], q: QueryContext) -> Dict[tuple, list]:
    out = {}
    for k, row in table.items():
        out[k] = [len(v) if agg.op == AggOp.DISTINCTCOUNT else v for v, agg in zip(row, q.aggregations)]
    return out


def _close(a: float, b: float, exact: bool) -> bool:
    if a == b:
        return True
    if exact:
        return False
    return abs(a - b) <= REL_TOL * max(abs(a), abs(b))


def assert_rows_equal(got: Dict[tuple, list], exp: Dict[tuple, list], q: QueryContext, exact_float=True, what="", sums=True):
    """sums=False: the SUM / AVG values are left to assert_matches_reference (tests/reference.py); AVG counts are compared"""
    assert set(got.keys()) == set(exp.keys()), f"{what}: group sets differ: {len(got)} vs {len(exp)}; " \
        f"missing={list(set(exp) - set(got))[:3]} extra={list(set(got) - set(exp))[:3]}"
    for k, erow in exp.items():
        grow = got[k]
        for a, agg in enumerate(q.aggregations):
            if grow[a] is None or erow[a] is None:
                assert grow[a] is None and erow[a] is None, f"{what}: {k} {agg}: {grow[a]!r} != {erow[a]!r} (SQL NULL)"
            elif agg.op == AggOp.AVG:
                assert grow[a][1] == erow[a][1], f"{what}: {k} {agg}: count {grow[a][1]} != {erow[a][1]}"
                assert not sums or _close(grow[a][0], erow[a][0], exact_float), f"{what}: {k} {agg}: sum {grow[a][0]!r} != {erow[a][0]!r}"
            elif agg.op in (AggOp.COUNT, AggOp.DISTINCTCOUNT):
                assert grow[a] == erow[a], f"{what}: {k} {agg}: {grow[a]} != {erow[a]}"
            else:
                ex = exact_float or agg.op in (AggOp.MIN, AggOp.MAX)
                assert (not sums and agg.op == AggOp.SUM) or _close(grow[a], erow[a], ex), f"{what}: {k} {agg}: {grow[a]!r} != {erow[a]!r}"


def reference_of(segments, q):
    """(per-segment, merged) reference results of q over the segments' decoded columns, or None where the reference cannot
    evaluate the query: chunk-compressed raw columns (their source values are not held here), null handling (enableNullHandling,
    IS [NOT] NULL), and the ORDER BY trim (it drops groups)"""
    if getattr(q, "null_handling", False) or q.trim(True)[0] > 0 or q.trim(False)[0] > 0:
        return None
    preds = filter_predicates(q.filter) + [p for a in q.aggregations for p in filter_predicates(a.filter)]
    if any(p.type in (PredicateType.IS_NULL, PredicateType.IS_NOT_NULL) for p in preds):
        return None
    cols = set(q.group_by) | {a.column for a in q.aggregations if a.column} | {p.column for p in preds}
    if any(reference.raw_is_compressed(s.columns[c]) for s in segments for c in cols if c in s.columns):
        return None
    srcs = [reference.SegmentSource(s) for s in segments]
    cols = cols or {next(c for c, ci in segments[0].columns.items() if not reference.raw_is_compressed(ci))}   # (the doc count)
    return [reference.reference(s, q) for s in srcs], reference.reference(reference.concat(srcs, cols), q)


def filter_predicates(node) -> list:
    if node is None:
        return []
    if isinstance(node, (And, Or)):
        return [p for ch in node.children for p in filter_predicates(ch)]
    if isinstance(node, Not):
        return filter_predicates(node.child)
    return [node]


def check_query(segments, sql_or_q, group=None, flags_list=(0,), exact_float=True, check_combined=True, check_stats=True):
    """Run per-segment and combined on the device and compare with the oracle, and with tests/reference.py where it can
    evaluate the query (its bound then replaces the relative tolerance of float SUM / AVG).  Returns the last native Result."""
    q = parse_sql(sql_or_q) if isinstance(sql_or_q, str) else sql_or_q
    own = group is None
    if own:
        staged = [native.StagedSegment(s) for s in segments]
        group = native.SegmentGroup(staged)
    orc = [oracle.execute(s, q) for s in segments]
    ref = reference_of(segments, q)
    # a table that reached numGroupsLimit has dropped groups: the reference does not apply, the oracle's sums stay checked
    use_ref = lambda t: ref is not None and t.stats["num_groups_limit_reached"] == 0
    last = None
    for flags in flags_list:
        res = native.execute(group, q, flags)
        assert len(res.tables) == len(segments)
        for i, (t, o) in enumerate(zip(res.tables, orc)):
            assert_rows_equal(t.rows(), oracle_rows(o), q, exact_float, what=f"segment {i} flags={flags}", sums=exact_float or not use_ref(t))
            if use_ref(t):
                reference.assert_matches_reference(t.rows(), ref[0][i], q, what=f"segment {i} flags={flags} vs reference")
            for key in ("num_docs_scanned", "num_entries_scanned_post_filter", "num_total_docs") if check_stats else ("num_total_docs",):
                assert t.stats[key] == o.stats[key], f"segment {i}: {key}: {t.stats[key]} != {o.stats[key]}"
            # DISTINCTCOUNT value sets (intermediate result) as dictId sets
            for a, agg in enumerate(q.aggregations):
                if agg.op == AggOp.DISTINCTCOUNT:
                    keys_n = t.keys() if q.group_by else [()]
                    keys_o = o.decoded_keys() if q.group_by else [()]
                    off_n, ids_n = t.distinct[a]
                    off_o, ids_o = o.distinct[a]
                    sets_o = {k: ids_o[off_o[g]:off_o[g + 1]].tolist() for g, k in enumerate(keys_o)}
                    for g, k in enumerate(keys_n):
                        assert ids_n[off_n[g]:off_n[g + 1]].tolist() == sets_o[k], f"segment {i}: distinct set of {k}"
        res.free()
        if check_combined:
            res = native.execute(group, q, flags | native.PB_Q_COMBINE)
            assert len(res.tables) == 1
            exp = combined_rows(oracle.combine(orc), q)
            assert_rows_equal(res.tables[0].rows(), exp, q, exact_float, what=f"combined flags={flags}", sums=exact_float or not use_ref(res.tables[0]))
            if use_ref(res.tables[0]):
                reference.assert_matches_reference(res.tables[0].rows(), ref[1], q, what=f"combined flags={flags} vs reference")
            assert not check_stats or res.tables[0].stats["num_docs_scanned"] == sum(o.stats["num_docs_scanned"] for o in orc)
            assert res.tables[0].stats["num_total_docs"] == sum(s.num_docs for s in segments)
            last = res
    if own:
        group.release()
        for s in staged:
            s.release()
    return last
