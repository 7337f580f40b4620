"""The two device paths that decide which groups come back -- numGroupsLimit (first docs + pb_select_first_kernel on dense
per-segment tables, tickets on hash tables) and the ORDER BY ... LIMIT trim (pb_order_key_kernel, the radix select, the
okey filter of pb_finalize_kernel) -- held to the exact reference (tests/reference.py: limit_reference,
assert_trim_matches_reference): a seeded fuzz over the fuzz tables and deterministic cases at the edges.

PB_FUZZ_SEEDS="0,2" narrows the fuzz seeds."""
import os

import numpy as np
import pytest

from oracle import oracle
from pinot_b200 import native
from pinot_b200.query import parse_sql
from pinot_b200.segment_writer import DataType, build_column, make_segment
from tests import fuzz_gen
from tests.reference import Col, assert_trim_matches_reference, concat, limit_reference, order_double

SEEDS = [int(s) for s in os.environ["PB_FUZZ_SEEDS"].split(",")] if os.environ.get("PB_FUZZ_SEEDS") else [0, 1, 2, 3]
QUERIES_PER_SEED = 5
FLAGS = (0, native.PB_Q_GENERIC_KERNEL, native.PB_Q_NO_TMA)
DENSE, HASH = 1, 2


@pytest.fixture(scope="module", autouse=True)
def _device():
    native.init()


def _group(segs):
    staged = [native.StagedSegment(s) for s in segs]
    return staged, native.SegmentGroup(staged)


def _release(staged, g):
    g.release()
    for s in staged:
        s.release()


def _key_space(seg, q):
    return int(np.prod([seg.columns[c].cardinality for c in q.group_by], dtype=object))


def check_table(t, lref, q, combined, what):
    """one result table against limit_reference + the trim"""
    rows, flag = t.rows(), t.stats["num_groups_limit_reached"]
    assert lref.reached is None or flag == int(lref.reached), f"{what}: num_groups_limit_reached {flag}, expected {int(lref.reached)}"
    assert len(rows) <= lref.at_most, f"{what}: {len(rows)} groups > numGroupsLimit {lref.at_most}"
    assert_trim_matches_reference(rows, lref.rows, q, combined, what, complete=lref.exact or not flag)
    return rows


def run_and_check(group, segs, srcs, sql, what, per_segment=True, replays=0, flags_list=FLAGS):
    """per segment and combined under each flag set; `replays` more combined runs under flags 0 (the plan cache, then its
    CUDA graph).  Returns the plan_info of every call."""
    q = parse_sql(sql)
    orc = [oracle.execute(s, q) for s in segs]
    plans = []
    for flags in flags_list:
        if per_segment:
            res = native.execute(group, q, flags)
            plans.append(res.plan_info)
            mode = res.plan_info["table_mode"]
            for i, (t, o, seg, src) in enumerate(zip(res.tables, orc, segs, srcs)):
                w = f"{what} flags={flags} segment {i}: {sql}"
                lref = limit_reference(src, q, "hash" if mode == HASH else "dense", _key_space(seg, q))
                check_table(t, lref, q, False, w)
                for key in ("num_docs_scanned", "num_entries_scanned_post_filter", "num_total_docs"):
                    assert t.stats[key] == o.stats[key], f"{w}: {key}: {t.stats[key]} != {o.stats[key]}"
                if mode == DENSE:        # (the oracle's key generator is Pinot's: doc order)
                    assert t.stats["num_groups_limit_reached"] == o.stats["num_groups_limit_reached"], w
            res.free()
        for rep in range(1 + (replays if flags == 0 else 0)):
            res = native.execute(group, q, flags | native.PB_Q_COMBINE)
            plans.append(res.plan_info)
            mode = res.plan_info["table_mode"]
            w = f"{what} flags={flags} combined (run {rep}): {sql}"
            m = "hash" if mode == HASH else "dense" if len(segs) == 1 else "merged"
            lref = limit_reference(concat(srcs), q, m, _key_space(segs[0], q))
            t = res.tables[0]
            check_table(t, lref, q, True, w)
            assert t.stats["num_docs_scanned"] == sum(o.stats["num_docs_scanned"] for o in orc), w
            assert t.stats["num_total_docs"] == sum(s.num_docs for s in segs), w
            res.free()
    return plans


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_shaped_fuzz_against_reference(seed):
    segs, srcs, _ = fuzz_gen.make_tables(seed)
    staged, g = _group(segs)
    rng = np.random.default_rng(1_000 + seed)
    try:
        for qi in range(QUERIES_PER_SEED):
            sql = fuzz_gen.make_shaped_query(rng, srcs[0])
            per_seg = not ("kwa" in sql.split("GROUP BY")[-1] and len(segs) > 3)
            run_and_check(g, segs, srcs, sql, f"seed {seed} query {qi}", per_segment=per_seg, replays=3 if qi == 0 else 0)
    finally:
        _release(staged, g)


# ---- deterministic cases ----

def _table(name, n, cols):
    """cols: name -> (DataType, values, has_dictionary)"""
    seg = make_segment(name, [build_column(c, dt, v, dictionary=d) for c, (dt, v, d) in cols.items()])
    src = {c: Col(np.asarray(v).astype(np.float64 if dt in (DataType.FLOAT, DataType.DOUBLE) else np.int64)
                  if dt != DataType.STRING else np.array(v, dtype="S"), dt, d) for c, (dt, v, d) in cols.items()}
    return seg, src


def _run(segs, srcs, sql, what, **kw):
    staged, g = _group(segs)
    try:
        return run_and_check(g, segs, srcs, sql, what, **kw)
    finally:
        _release(staged, g)


def _limit_table(n=20_000, groups=200, seed=3):
    """dict key k of `groups` values whose first docs come in an order unrelated to their values or sums; v > 0, f 0/1"""
    r = np.random.default_rng(seed)
    k = r.integers(0, groups, n)
    k[:groups] = r.permutation(groups)
    v = r.integers(1, 1000, n)
    return _table("lim", n, {"k": (DataType.INT, k.astype(np.int32), True), "v": (DataType.INT, v.astype(np.int32), True),
                             "f": (DataType.INT, r.integers(0, 2, n).astype(np.int32), True)})


@pytest.mark.gpu
def test_trim_ranks_only_the_groups_the_limit_admits():
    """defect 1: per segment, numGroupsLimit 50 of 200 keys and a trim to 10: the trim ranks the 50 admitted groups
    (Pinot limits the keys first, then trims), so exactly their 10 best come back"""
    seg, src = _limit_table()
    for tail in ("ORDER BY SUM(v) DESC LIMIT 1", "ORDER BY k ASC LIMIT 2", "ORDER BY COUNT(*) DESC LIMIT 1"):
        sql = f"SET numGroupsLimit = 50; SET minSegmentGroupTrimSize = 10; SET minServerGroupTrimSize = 10; SET groupTrimThreshold = 20; " \
              f"SELECT k, SUM(v), COUNT(*) FROM t WHERE f = 0 GROUP BY k {tail}"
        _run([seg], [src], sql, "limit then trim", replays=3)


@pytest.mark.gpu
def test_limit_flag_survives_the_trim():
    """defect 2: the flag comes from the group count before the trim -- a dense table limited to 50 groups and trimmed to
    10, and a hash table holding exactly `limit` groups trimmed to 10"""
    seg, src = _limit_table()
    sql = "SET numGroupsLimit = 50; SET minSegmentGroupTrimSize = 10; SET minServerGroupTrimSize = 10; SET groupTrimThreshold = 20; " \
          "SELECT k, SUM(v) FROM t GROUP BY k ORDER BY SUM(v) DESC LIMIT 1"
    _run([seg], [src], sql, "dense flag")
    r = np.random.default_rng(8)
    n = 5_000
    rk = r.integers(0, 100, n) * 1_000_003
    seg, src = _table("hlim", n, {"rk": (DataType.LONG, rk, False), "v": (DataType.INT, r.integers(0, 50, n).astype(np.int32), True)})
    sql = "SET numGroupsLimit = 100; SET minSegmentGroupTrimSize = 10; SET minServerGroupTrimSize = 10; SET groupTrimThreshold = 20; " \
          "SELECT rk, SUM(v), COUNT(*) FROM t GROUP BY rk ORDER BY COUNT(*) DESC LIMIT 1"
    plans = _run([seg], [src], sql, "hash flag")
    assert all(p["table_mode"] == HASH for p in plans), plans


@pytest.mark.gpu
def test_empty_aggregates_rank_as_their_final_results():
    """defects 3 and 4 at the cut: a filtered AVG without input ranks as -inf (AvgAggregationFunction's DEFAULT_FINAL_RESULT),
    below every real (here negative) average; MIN / MAX without input (all inputs NaN, or none through the FILTER clause)
    rank as the +inf / -inf they report, tied with groups that hold a real +inf / -inf"""
    n, groups = 12_000, 30
    r = np.random.default_rng(21)
    k = np.arange(n) % groups
    f = np.where(k < 10, 0, r.integers(0, 2, n))               # groups 0-9: no doc with f = 1
    v = -r.integers(1, 1000, n)
    x = np.where(k < 10, np.nan, np.where(k < 20, np.inf, r.normal(0, 5, n)))
    y = np.where(k < 10, np.nan, np.where(k < 20, -np.inf, r.normal(0, 5, n)))
    seg, src = _table("empty", n, {"k": (DataType.INT, k.astype(np.int32), True), "f": (DataType.INT, f.astype(np.int32), True),
                                   "v": (DataType.INT, v.astype(np.int32), True), "x": (DataType.DOUBLE, x, False),
                                   "y": (DataType.DOUBLE, y, False)})
    opts = "SET minSegmentGroupTrimSize = 5; SET minServerGroupTrimSize = 5; SET groupTrimThreshold = 10; "
    for tail in ("ORDER BY AVG(v) FILTER(WHERE f = 1) ASC LIMIT 1", "ORDER BY MIN(x) DESC LIMIT 1", "ORDER BY MAX(y) ASC LIMIT 1",
                 "ORDER BY MIN(v) FILTER(WHERE f = 1) DESC LIMIT 1", "ORDER BY MAX(v) FILTER(WHERE f = 1) ASC LIMIT 1"):
        sql = opts + "SELECT k, AVG(v) FILTER(WHERE f = 1), MIN(x), MAX(y), MIN(v) FILTER(WHERE f = 1), MAX(v) FILTER(WHERE f = 1), " \
                     f"COUNT(*) FROM t GROUP BY k {tail}"
        _run([seg], [src], sql, "empty aggregates", replays=3)


@pytest.mark.gpu
def test_ties_at_the_cut_are_kept():
    """40 groups of exactly 100 docs and 10 of 50: a trim to 10 by COUNT keeps all 40 tied groups, and no smaller one"""
    k = np.concatenate([np.repeat(np.arange(40), 100), np.repeat(np.arange(40, 50), 50)])
    k = np.random.default_rng(4).permutation(k)
    seg, src = _table("ties", len(k), {"k": (DataType.INT, k.astype(np.int32), True)})
    for d in ("DESC", "ASC"):
        sql = "SET minSegmentGroupTrimSize = 10; SET minServerGroupTrimSize = 10; SET groupTrimThreshold = 20; " \
              f"SELECT k, COUNT(*) FROM t GROUP BY k ORDER BY COUNT(*) {d} LIMIT 1"
        _run([seg], [src], sql, f"ties {d}")


@pytest.mark.gpu
def test_group_counts_at_the_trim_size_and_threshold():
    """exactly size, size +- 1, threshold and threshold + 1 groups (size 10, combined threshold 25): distinct sums"""
    for groups in (9, 10, 11, 25, 26):
        n = groups * 7
        k = np.arange(n) % groups
        v = k * 3 + 1
        seg, src = _table(f"g{groups}", n, {"k": (DataType.INT, k.astype(np.int32), True), "v": (DataType.LONG, v.astype(np.int64), True)})
        sql = "SET minSegmentGroupTrimSize = 10; SET minServerGroupTrimSize = 10; SET groupTrimThreshold = 25; " \
              "SELECT k, SUM(v) FROM t GROUP BY k ORDER BY SUM(v) DESC LIMIT 1"
        _run([seg], [src], sql, f"{groups} groups")


def _raw_key_table(n=30_000, seed=6):
    r = np.random.default_rng(seed)
    rki, rkj = r.integers(-40, 40, n), r.integers(-3, 3, n)
    rki[::97], rkj[::97] = -1, -1                              # the all-ones key pattern of two 32-bit fields
    return _table("rawk", n, {"k3": (DataType.INT, r.integers(0, 3, n).astype(np.int32), True),
                              "rki": (DataType.INT, rki.astype(np.int32), False), "rkj": (DataType.INT, rkj.astype(np.int32), False),
                              "m": (DataType.LONG, r.integers(-10**6, 10**6, n), True)})


@pytest.mark.gpu
def test_raw_key_fields_order_signed_across_key_words_and_at_the_sentinel():
    """ORDER BY rkj over keys k3, rki, rkj (66 bits: rkj's field crosses into the second key word); ORDER BY rki / rkj over
    rki, rkj, whose key -1, -1 is the all-ones sentinel; negative values of raw INT fields order below positive ones"""
    seg, src = _raw_key_table()
    opts = "SET minSegmentGroupTrimSize = 10; SET minServerGroupTrimSize = 10; SET groupTrimThreshold = 20; "
    for sql in ("SELECT k3, rki, rkj, COUNT(*), SUM(m) FROM t GROUP BY k3, rki, rkj ORDER BY rkj DESC LIMIT 1",
                "SELECT k3, rki, rkj, COUNT(*), SUM(m) FROM t GROUP BY k3, rki, rkj ORDER BY rkj ASC LIMIT 1",
                "SELECT rki, rkj, COUNT(*), MAX(m) FROM t GROUP BY rki, rkj ORDER BY rki DESC LIMIT 2",
                "SELECT rki, rkj, COUNT(*), MAX(m) FROM t GROUP BY rki, rkj ORDER BY rkj ASC LIMIT 2",
                "SELECT rki, rkj, COUNT(*), MAX(m) FROM t GROUP BY rki, rkj ORDER BY COUNT(*) DESC LIMIT 2",
                # the all-ones key (doc 0) under a reachable limit takes a ticket like any other key
                "SET numGroupsLimit = 3; SELECT rki, rkj, COUNT(*), SUM(m) FROM t GROUP BY rki, rkj ORDER BY rki DESC LIMIT 1",
                "SET numGroupsLimit = 1; SELECT rki, rkj, COUNT(*) FROM t GROUP BY rki, rkj LIMIT 10"):
        plans = _run([seg], [src], opts + sql, "raw keys")
        assert all(p["table_mode"] == HASH for p in plans), plans


def _double_key_rows(t):
    """{key bits (NaN canonical): COUNT} of a single raw FLOAT / DOUBLE key (a dict keyed by float folds -0.0 into 0.0)"""
    keys = t.key_values[0].astype(np.float64)
    return {order_double(float(x)): int(c) for x, c in zip(keys, t.longs[0])}


@pytest.mark.gpu
def test_raw_floating_keys_order_by_double_compare():
    """raw DOUBLE key holding -0.0, 0.0, +-inf and NaN, and a raw FLOAT key with negative values: Double.compare order,
    -0.0 below 0.0, NaN above +inf"""
    vals = np.array([-np.inf, -2.5, -1.0, -0.0, 0.0, 0.5, 3.0, 1e300, np.inf, np.nan])
    fvals = np.array([-7.5, -3.25, -1.0, -0.125, 0.25, 2.0, 9.5, 100.0], dtype=np.float32)
    n = 4_000
    r = np.random.default_rng(2)
    d = vals[np.arange(n) % len(vals)]
    fl = fvals[r.integers(0, len(fvals), n)]
    seg, src = _table("fkeys", n, {"d": (DataType.DOUBLE, d, False), "fl": (DataType.FLOAT, fl, False)})
    counts = {order_double(float(x)): n // len(vals) for x in vals}
    staged, g = _group([seg])
    try:
        for col, pool in (("d", vals), ("fl", fvals.astype(np.float64))):
            for desc in (True, False):
                q = parse_sql("SET minSegmentGroupTrimSize = 3; SET minServerGroupTrimSize = 3; SET groupTrimThreshold = 6; "
                              f"SELECT COUNT(*) FROM t GROUP BY {col} ORDER BY {col} {'DESC' if desc else 'ASC'} LIMIT 1")
                ranks = sorted((order_double(float(x)) for x in pool), reverse=desc)
                for flags in (0, native.PB_Q_COMBINE):
                    size, thr = q.trim(bool(flags))    # per segment 5 of 10 / 8 groups; combined: no trim at <= 10
                    want = set(ranks) if len(ranks) <= thr else set(ranks[:size])
                    res = native.execute(g, q, flags)
                    got = _double_key_rows(res.tables[0])
                    assert set(got) == want, (col, desc, flags, sorted(got), sorted(want))
                    if col == "d":
                        assert all(got[k] == counts[k] for k in got), (got, counts)
                    res.free()
    finally:
        _release(staged, g)


@pytest.mark.gpu
def test_long_sums_that_differ_in_the_low_byte():
    """40 groups whose SUMs are one LONG value just below 2^53 plus 0..39: the order keys differ only in their last radix
    digit, so each of the 8 passes decides"""
    base = (1 << 53) - 4096                        # one doc per group: every sum is exact
    groups = 40
    k = np.arange(groups)
    v = base + k
    seg, src = _table("lowbyte", len(k), {"k": (DataType.INT, k.astype(np.int32), True), "v": (DataType.LONG, v.astype(np.int64), True)})
    for d in ("DESC", "ASC"):
        sql = "SET minSegmentGroupTrimSize = 7; SET minServerGroupTrimSize = 7; SET groupTrimThreshold = 14; " \
              f"SELECT k, SUM(v), COUNT(*) FROM t GROUP BY k ORDER BY SUM(v) {d} LIMIT 1"
        _run([seg], [src], sql, f"low byte {d}")


@pytest.mark.gpu
def test_trim_and_limit_on_a_2_pow_24_slot_dense_table():
    """4096 x 4096 dense slots (past 2^20: the hand-back counts the surviving groups first, pb_count_groups_kernel), with
    a trim, and with a numGroupsLimit below the key space as well"""
    n = 200_000
    r = np.random.default_rng(13)
    a, b = r.integers(0, fuzz_gen.WIDE, n), r.integers(0, fuzz_gen.WIDE, n)
    a[:2], b[:2] = [0, fuzz_gen.WIDE - 1], [fuzz_gen.WIDE - 1, 0]
    cols, src = [], {}
    for name, ids in (("ka", a), ("kb", b)):
        dv = np.arange(fuzz_gen.WIDE, dtype=np.int64) * 2
        cols.append(fuzz_gen._dict_col(name, DataType.INT, dv, ids))
        src[name] = fuzz_gen._src(DataType.INT, dv, ids)
    m = r.integers(-1000, 1000, n)
    cols.append(build_column("m", DataType.INT, m.astype(np.int32)))
    src["m"] = Col(m, DataType.INT)
    seg = make_segment("wide", cols)
    opts = "SET minSegmentGroupTrimSize = 50; SET minServerGroupTrimSize = 50; SET groupTrimThreshold = 100; "
    for pre in ("", "SET numGroupsLimit = 5000; "):
        for tail in ("ORDER BY SUM(m) DESC LIMIT 3", "ORDER BY kb ASC LIMIT 3"):
            plans = _run([seg], [src], pre + opts + f"SELECT ka, kb, SUM(m), COUNT(*) FROM t GROUP BY ka, kb {tail}", "2^24 slots",
                         flags_list=(0,), replays=1)
            assert all(p["table_mode"] == DENSE for p in plans), plans


@pytest.mark.gpu
def test_num_groups_limit_edges_on_each_aggregation_kernel():
    """numGroupsLimit 1, groups - 1, groups and key space - 1 on the general kernel and the rows kernel (a limit below the
    key space tracks first docs, which rules out the CTA-private table), and the key space itself on the CTA-table
    kernel, with and without a trim.  A query with a reachable limit is never fused."""
    n = 30_000
    r = np.random.default_rng(17)
    kk = r.integers(0, 60, n)                      # 60 of the 64 dictionary entries occur in the filtered docs
    kk[0] = 63                                     # (one more, filtered out: the dictionary keeps 64 entries)
    dv = np.arange(64, dtype=np.int64) * 7
    f = r.integers(0, 2, n)
    f[0] = 1
    v = r.integers(-500, 500, n)
    cols = [fuzz_gen._dict_col("k", DataType.INT, dv, kk),
            build_column("f", DataType.INT, f.astype(np.int32)), build_column("v", DataType.INT, v.astype(np.int32))]
    src = {"k": fuzz_gen._src(DataType.INT, dv, kk), "f": Col(f, DataType.INT), "v": Col(v, DataType.INT)}
    seg = make_segment("edges", cols)
    groups = len(np.unique(kk[f == 0]))
    seen = {}
    for limit in (1, groups - 1, groups, 63, 64):
        for body in ("SELECT k, SUM(v), COUNT(*) FROM t WHERE f = 0 GROUP BY k",                        # rows kernel
                     "SELECT k, SUM(v), COUNT(*) FILTER(WHERE v < 0) FROM t WHERE f = 0 GROUP BY k",    # no rows kernel (FILTER)
                     "SELECT k, MIN(v), MAX(v) FROM t WHERE f = 0 OR v > 400 GROUP BY k"):
            for tail in ("", " ORDER BY SUM(v) DESC LIMIT 1" if "SUM" in body else " ORDER BY k DESC LIMIT 1"):
                sql = f"SET numGroupsLimit = {limit}; SET minSegmentGroupTrimSize = 8; SET minServerGroupTrimSize = 8; " \
                      f"SET groupTrimThreshold = 16; {body}{tail}"
                plans = _run([seg], [src], sql, f"limit {limit}", replays=3 if limit == 1 else 0)
                for p in plans:
                    seen.setdefault(p["agg_kernel"], set()).add(limit)
                    assert not (limit < 64 and p["fused_agg"]), (sql, p)
    assert {1, 3} <= {a for a, ls in seen.items() if min(ls) < 64}, seen     # general and rows kernels under a reachable limit
    assert os.environ.get("PB_AGG_SMEM", "1") == "0" or 64 in seen.get(2, ()), seen
