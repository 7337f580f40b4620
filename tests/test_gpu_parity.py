"""Parity of the CUDA path (called through the C ABI) against the oracle and the reference's goldens.  -m gpu."""
import numpy as np
import pytest

from pinot_b200 import datagen, native
from pinot_b200.query import parse_sql
from pinot_b200.segment_writer import DataType, build_column, build_dict_column, make_segment
from tests.fixtures import FILTER, sv_segment
from oracle import oracle
from tests.parity import assert_rows_equal, check_query, combined_rows, oracle_rows

pytestmark = pytest.mark.gpu

AGG = "SELECT COUNT(*), SUM(column1), MAX(column3), MIN(column6), AVG(column7) FROM testTable"
ALL_FLAGS = (0, native.PB_Q_GENERIC_KERNEL, native.PB_Q_NO_TMA)


@pytest.fixture(scope="module")
def sv_group():
    native.init()
    seg = sv_segment()
    staged = [native.StagedSegment(seg) for _ in range(4)]
    g = native.SegmentGroup(staged)
    yield seg, g
    g.release()


def _row(res_table, key=()):
    return res_table.rows()[key]


def test_golden_aggregation_only(sv_group):   # InnerSegmentAggregationSingleValueQueriesTest.java:43-60
    seg, g = sv_group
    r = native.execute(g, parse_sql(AGG))
    row = _row(r.tables[0])
    assert (row[0], int(row[1]), int(row[2]), int(row[3]), int(row[4][0]), row[4][1]) == \
        (30000, 32317185437847, 2147419555, 1689277, 28175373944314, 30000)
    st = r.tables[0].stats
    assert (st["num_docs_scanned"], st["num_entries_scanned_post_filter"], st["num_total_docs"]) == (30000, 120000, 30000)
    r = native.execute(g, parse_sql(AGG + FILTER))
    row = _row(r.tables[0])
    assert (row[0], int(row[1]), int(row[2]), int(row[3]), int(row[4][0]), row[4][1]) == \
        (6129, 6875947596072, 999813884, 1980174, 4699510391301, 6129)
    st = r.tables[0].stats
    assert (st["num_docs_scanned"], st["num_entries_scanned_post_filter"], st["num_total_docs"]) == (6129, 24516, 30000)
    # 4 identical segments merged on the device == InterSegment goldens (x4)
    r = native.execute(g, parse_sql(AGG + FILTER), native.PB_Q_COMBINE)
    row = _row(r.tables[0])
    assert (row[0], int(row[1]), int(row[2]), int(row[3])) == (24516, 4 * 6875947596072, 999813884, 1980174)


@pytest.mark.parametrize("group_by,key,exp,key_f,exp_f", [
    (" GROUP BY column9", (11270,), (1, 815409257, 1215316262, 1328642550, 788414092, 1),
     (242920,), (3, 4348938306, 407993712, 296467636, 5803888725, 3)),
    (" GROUP BY column9, column11, column12", (1813102948, b"P", b"HEuxNvH"),
     (4, 2062187196, 1988589001, 394608493, 4782388964, 4),
     (1176631727, b"P", b"KrNxpdycSiwoRohEiTIlLqDHnx"), (1, 716185211, 489993380, 371110078, 487714191, 1)),
    (" GROUP BY column1, column6, column9, column11, column12",
     (484569489, 16200443, 1159557463, b"P", b"MaztCmmxxgguBUxPti"), (2, 969138978, 995355481, 16200443, 2222394270, 2),
     (1318761745, 353175528, 1172307870, b"P", b"HEuxNvH"), (2, 2637523490, 557154208, 353175528, 2427862396, 2)),
])
def test_golden_group_by(sv_group, group_by, key, exp, key_f, exp_f):   # :96-152
    seg, g = sv_group
    for sql, k, e in ((AGG + group_by, key, exp), (AGG + FILTER + group_by, key_f, exp_f)):
        r = native.execute(g, parse_sql(sql))
        row = _row(r.tables[0], k)
        assert (row[0], int(row[1]), int(row[2]), int(row[3]), int(row[4][0]), row[4][1]) == e


VERY_LARGE = " GROUP BY column1, column3, column6, column7, column9, column11, column12, column17, column18"


def test_golden_very_large_group_by(sv_group):   # :156-174 — the ARRAY_MAP holder's key space (> 64 bits of dictIds): 128-bit keys
    seg, g = sv_group
    for sql, k, e, st_e in (
            (AGG + VERY_LARGE, (1784773968, 204243323, 628170461, 1985159279, 296467636, b"P", b"HEuxNvH", 402773817, 2047180536),
             (1, 1784773968, 204243323, 628170461, 1985159279, 1), (30000, 0, 270000, 30000)),
            (AGG + FILTER + VERY_LARGE, (1361199163, 178133991, 296467636, 788414092, 1719301234, b"P", b"MaztCmmxxgguBUxPti", 1284373442, 752388855),
             (1, 1361199163, 178133991, 296467636, 788414092, 1), (6129, 63064, 55161, 30000))):
        r = native.execute(g, parse_sql(sql))
        row = _row(r.tables[0], k)
        assert (row[0], int(row[1]), int(row[2]), int(row[3]), int(row[4][0]), row[4][1]) == e
        st = r.tables[0].stats
        assert (st["num_docs_scanned"], st["num_entries_scanned_post_filter"], st["num_total_docs"]) == (st_e[0], st_e[2], st_e[3])
    check_query([seg, seg], AGG + FILTER + VERY_LARGE, flags_list=ALL_FLAGS)
    check_query([seg, seg], "SELECT COUNT(*), DISTINCTCOUNT(column5) FROM testTable" + VERY_LARGE)


def test_group_key_wider_than_128_bits_declines(sv_group):   # plan maker declines: PB_ERR_UNSUPPORTED, never a CPU fallback
    seg, g = sv_group
    # exactly 128 bits of dictIds (15 columns) still runs
    check_query([seg], "SELECT COUNT(*), SUM(column1) FROM testTable" + FILTER + VERY_LARGE + ", column5, daysSinceEpoch, column1, column3, column6, column7")
    q = parse_sql("SELECT COUNT(*) FROM testTable" + VERY_LARGE + ", column5, daysSinceEpoch, column1, column3, column6, column7, column9")   # 139 bits
    with pytest.raises(native.PinotB200Error) as ei:
        native.execute(g, q)
    assert ei.value.code == -2


def test_golden_inter_segment(sv_group):   # InterSegmentAggregationSingleValueQueriesTest.java:47-258
    seg, g = sv_group
    C = native.PB_Q_COMBINE
    assert _row(native.execute(g, parse_sql("SELECT COUNT(*) FROM testTable"), C).tables[0])[0] == 120000
    assert _row(native.execute(g, parse_sql("SELECT COUNT(*) FROM testTable" + FILTER), C).tables[0])[0] == 24516
    t = native.execute(g, parse_sql("SELECT COUNT(*) FROM testTable GROUP BY column9"), C).tables[0]
    assert max(v[0] for v in t.rows().values()) == 64420
    t = native.execute(g, parse_sql("SELECT COUNT(*) FROM testTable" + FILTER + " GROUP BY column9"), C).tables[0]
    assert max(v[0] for v in t.rows().values()) == 17080
    assert _row(native.execute(g, parse_sql("SELECT MAX(column1), MAX(column3) FROM testTable" + FILTER), C).tables[0]) == [2146952047.0, 999813884.0]
    assert _row(native.execute(g, parse_sql("SELECT MIN(column1), MIN(column3) FROM testTable"), C).tables[0]) == [240528.0, 17891.0]
    dc = "SELECT DISTINCTCOUNT(column1), DISTINCTCOUNT(column3) FROM testTable"
    assert _row(native.execute(g, parse_sql(dc), C).tables[0]) == [6582, 21910]
    assert _row(native.execute(g, parse_sql(dc + FILTER), C).tables[0]) == [1872, 4556]
    t = native.execute(g, parse_sql(dc + " GROUP BY column9"), C).tables[0]
    assert (max(v[0] for v in t.rows().values()), max(v[1] for v in t.rows().values())) == (3495, 11961)
    t = native.execute(g, parse_sql(dc + FILTER + " GROUP BY column9"), C).tables[0]
    assert (max(v[0] for v in t.rows().values()), max(v[1] for v in t.rows().values())) == (1272, 3289)


def test_sv_segment_vs_oracle_all_kernels():
    seg = sv_segment()
    for sql in (AGG, AGG + FILTER, AGG + FILTER + " GROUP BY column9, column11",
                "SELECT COUNT(*), DISTINCTCOUNT(column17) FROM testTable WHERE column6 < 500000000 OR column11 NOT IN ('t','P') GROUP BY column12",
                "SELECT SUM(column18) FROM testTable WHERE NOT (column7 IN (1111197135, 296467636)) AND column17 <> 635942547",
                "SELECT COUNT(*) FROM testTable WHERE column5 = 'nope'",
                "SELECT COUNT(*), MIN(column1) FROM testTable WHERE daysSinceEpoch > 126164076 GROUP BY daysSinceEpoch"):
        check_query([seg, seg], sql, flags_list=ALL_FLAGS)


@pytest.fixture(scope="module")
def synth():
    native.init()
    segs = [datagen.make_segment_synth(i, n, vary_dim_dictionaries=(i > 0)) for i, n in enumerate((100_003, 65_536, 8_192 * 3 + 1))]
    staged = [native.StagedSegment(s) for s in segs]
    g = native.SegmentGroup(staged)
    yield segs, g
    g.release()


def test_config1_keyless_sum(synth):
    segs, g = synth
    check_query(segs, datagen.config1_sql(segs[0]), group=g, flags_list=ALL_FLAGS)


def test_config2_filter_group_by(synth):
    segs, g = synth
    check_query(segs, datagen.config2_sql(segs, 16), group=g, flags_list=ALL_FLAGS)
    check_query(segs, datagen.config2_sql(segs, 500), group=g, flags_list=(0,))


def test_config3_inverted_index_and_or(synth):
    segs, g = synth
    d1 = segs[0].columns["c1"].dictionary_values()
    d3 = segs[0].columns["c3"].dictionary_values()
    d0 = segs[0].columns["d0"].dictionary_values()
    sql = (f"SELECT d0, d1, d2, d3, d4, SUM(m0), COUNT(*), MIN(m1), MAX(m2) FROM t WHERE (c1 IN ({', '.join(str(int(v)) for v in d1[:8])}) "
           f"OR c3 = {int(d3[5])}) AND d0 IN ({int(d0[1])}, {int(d0[6])}) GROUP BY d0, d1, d2, d3, d4 LIMIT 100000")
    check_query(segs, sql, group=g, flags_list=(0, native.PB_Q_GENERIC_KERNEL))


def test_config4_string_key_distinct_raw_double(synth):
    segs, g = synth
    d2 = segs[0].columns["c2"].dictionary_values()
    sql = f"SELECT s0, DISTINCTCOUNT(c0), SUM(x0), AVG(x1) FROM t WHERE c2 < {int(d2[len(d2) // 2])} GROUP BY s0 LIMIT 100000"
    check_query(segs, sql, group=g, exact_float=False)


def test_config5_raw_long_key_hash(synth):
    segs, g = synth
    check_query(segs, "SET numGroupsLimit = 20000000; SELECT k0, SUM(m0), COUNT(*) FROM t GROUP BY k0 LIMIT 100000000", group=g)


def test_sorted_column_and_raw_predicates(synth):
    segs, g = synth
    check_query(segs, "SELECT t0, COUNT(*), MAX(m0) FROM t WHERE t0 BETWEEN 20010 AND 20040 AND x0 < 0.5 GROUP BY t0", group=g)
    check_query(segs, "SELECT COUNT(*), SUM(x1), MIN(x0), MAX(k0) FROM t WHERE k0 > 5000000000000 AND t0 <> 20003", group=g, exact_float=False)
    check_query(segs, "SELECT c5, c6, COUNT(*) FROM t WHERE t0 IN (20001, 20005, 20006, 20050) OR c7 = 0 GROUP BY c5, c6", group=g)


def test_empty_and_match_all(synth):
    segs, g = synth
    check_query(segs, "SELECT COUNT(*), SUM(m0), MIN(m1), MAX(m2) FROM t WHERE c1 < -5", group=g)
    check_query(segs, "SELECT COUNT(*), SUM(m0), MIN(m1), MAX(m2) FROM t WHERE c1 > -5", group=g)
    check_query(segs, "SELECT d1, COUNT(*) FROM t WHERE c1 < -5 GROUP BY d1", group=g)


def test_gather_in_place_from_mapped_host_buffers(monkeypatch):
    """PB_Q_GATHER_IN_PLACE: group-by / aggregation columns of cold segments are read from the caller's page-locked
    buffers (no HBM copy) where that is cheaper than copying them; predicate columns are staged on the copy stream and
    the kernels follow in per-segment waves.  Row counts chosen so the bit streams end mid-word."""
    native.init()
    segs = [datagen.make_segment_synth(i, n, vary_dim_dictionaries=(i > 0)) for i, n in enumerate((150_001, 120_011, 100_003))]
    registered = []
    for s in segs:
        for c in s.columns.values():
            if c.forward_index is not None and c.forward_index.nbytes:
                native.host_register(c.forward_index)
                registered.append(c.forward_index)
    d1 = segs[0].columns["c1"].dictionary_values()
    in3 = ", ".join(str(int(v)) for v in d1[10:13])
    d0v = int(segs[0].columns["d0"].dictionary_values()[3])
    try:
        for cost, sql, exact, min_cols in (
                (None, datagen.config2_sql(segs, 16), True, 3 * 3),          # cost rule: wide metric columns in place, narrow keys copied
                ("0", datagen.config2_sql(segs, 16), True, 6 * 3),           # forced: every gathered column in place
                ("0", f"SELECT s0, d3, DISTINCTCOUNT(c0), SUM(x0), MAX(k0) FROM t WHERE c1 IN ({in3}) GROUP BY s0, d3 LIMIT 100000", False, 5 * 3),
                ("0", f"SELECT d0, COUNT(*), SUM(m0) FROM t WHERE d0 = {d0v} AND c1 > 10 GROUP BY d0", True, 1 * 3),   # d0: predicate AND key
                ("0", "SELECT MIN(m1), MAX(m2), AVG(m0) FROM t", True, 3 * 3),
                (None, "SELECT d1, MIN(m1), MAX(m2), AVG(m0) FROM t WHERE c2 > 100 GROUP BY d1", True, 0)):   # unselective: everything is copied
            if cost is None:
                monkeypatch.delenv("PB_IN_PLACE_COST", raising=False)
            else:
                monkeypatch.setenv("PB_IN_PLACE_COST", cost)
            staged = [native.StagedSegment(s) for s in segs]       # cold: nothing resident yet
            g = native.SegmentGroup(staged)
            q = parse_sql(sql)
            r = native.execute(g, q, native.PB_Q_GATHER_IN_PLACE | native.PB_Q_COMBINE)
            assert r.in_place_columns >= min_cols, (sql, r.in_place_columns)
            if min_cols == 0:
                assert r.in_place_columns == 0
            rows_cold = r.tables[0].rows()       # computed in waves behind the staging copies
            cold_stats = dict(r.tables[0].stats)
            r.free()
            check_query(segs, q, group=g, flags_list=(native.PB_Q_GATHER_IN_PLACE,), exact_float=exact)
            r = native.execute(g, q, native.PB_Q_COMBINE)      # warm, single wave; same path check_query just verified
            assert_rows_equal(rows_cold, r.tables[0].rows(), q, exact, what="cold (waves) vs warm")
            assert cold_stats["num_docs_scanned"] == r.tables[0].stats["num_docs_scanned"]
            r.free()
            g.release()
            for st_ in staged:
                st_.release()
    finally:
        for a in registered:
            native.host_unregister(a)


@pytest.mark.parametrize("bits", list(range(1, 21)) + [24])
def test_every_bit_width(bits):
    """Forward index widths 1..20 and 24 through both predicate paths (range + IN) and the gather path."""
    native.init()
    rng = np.random.default_rng(bits)
    n = 40_000 + bits
    if bits == 1:
        card = 2
    elif bits < 17:
        card = (1 << bits) - 1
    else:
        card = (1 << (bits - 1)) + 5          # bitsPerElement = bit length of (card - 1)
    if bits <= 20:
        dvals = np.sort(rng.choice(max(card * 4, 64), size=card, replace=False)).astype(np.int32)
    else:
        dvals = (np.arange(card, dtype=np.int64) * 3).astype(np.int32)
    ids = rng.integers(0, card, n, dtype=np.uint32)
    k = min(card, n)
    ids[rng.choice(n, size=k, replace=False)] = rng.choice(card, size=k, replace=False).astype(np.uint32)
    ids[0] = card - 1
    col = build_dict_column("w", DataType.INT, dvals, ids)
    assert col.bits_per_element == bits
    g_ids = rng.integers(0, 7, n, dtype=np.uint32)
    gcol = build_dict_column("g", DataType.INT, np.arange(7, dtype=np.int32) * 11, g_ids)
    seg = make_segment(f"w{bits}", [col, gcol])
    lo, hi = int(dvals[card // 4]), int(dvals[(3 * card) // 4])
    pick = ", ".join(str(int(v)) for v in dvals[:: max(1, card // 9)][:9])
    for sql in (f"SELECT g, COUNT(*), SUM(w), MIN(w), MAX(w) FROM t WHERE w BETWEEN {lo} AND {hi} GROUP BY g",
                f"SELECT COUNT(*), SUM(w) FROM t WHERE w IN ({pick})",
                f"SELECT w, COUNT(*) FROM t WHERE w NOT IN ({pick}) AND g <> 11 GROUP BY w LIMIT 10000000"):
        check_query([seg], sql, flags_list=(0, native.PB_Q_GENERIC_KERNEL), check_combined=(bits <= 20))


def test_candidate_leaves_of_a_flat_conjunction():
    """Flat AND whose most selective leaf leaves <= 3 % of the docs (by dictionary statistics): the other scan leaves run
    on the candidates only, one lane per surviving doc, reading their forward index in place (DevLeaf::gather) — the
    device form of AndDocIdSet + SVScanDocIdIterator.applyAnd.  Covers dictionary range / IN (smem LUT and global
    bitset) / NOT IN, raw LONG and DOUBLE ranges, a raw IN, and a skewed column whose estimate is far off (the candidate
    list then takes several passes)."""
    native.init()
    rng = np.random.default_rng(7)
    n = 300_017
    # a: 1000 values, heavily skewed: 70 % of the docs carry dictId 3 (the statistics say 0.1 %)
    a_ids = rng.integers(0, 1000, n, dtype=np.uint32)
    a_ids[rng.random(n) < 0.7] = 3
    a_ids[:1000] = np.arange(1000, dtype=np.uint32)
    a = build_dict_column("a", DataType.INT, np.arange(1000, dtype=np.int32) * 7 + 1, a_ids)
    b_ids = rng.integers(0, 5000, n, dtype=np.uint32); b_ids[:5000] = np.arange(5000, dtype=np.uint32)
    b = build_dict_column("b", DataType.INT, np.arange(5000, dtype=np.int32) * 3, b_ids)
    c_ids = rng.integers(0, 20000, n, dtype=np.uint32); c_ids[:20000] = np.arange(20000, dtype=np.uint32)   # > 8192: bitset in global memory
    c = build_dict_column("c", DataType.LONG, np.arange(20000, dtype=np.int64) * 1_000_003, c_ids)
    d_ids = rng.integers(0, 6, n, dtype=np.uint32)
    d = build_dict_column("d", DataType.INT, np.arange(6, dtype=np.int32) + 10, d_ids)
    x = build_column("x", DataType.DOUBLE, rng.random(n), dictionary=False)
    k = build_column("k", DataType.LONG, rng.integers(0, 1_000_000, n, dtype=np.int64), dictionary=False)
    m = build_dict_column("m", DataType.INT, np.arange(50_000, dtype=np.int32) * 2,
                          np.concatenate([np.arange(50_000, dtype=np.uint32), rng.integers(0, 50_000, n - 50_000, dtype=np.uint32)]))
    seg = make_segment("cand", [a, b, c, d, x, k, m])
    seg2 = make_segment("cand2", [build_dict_column("a", DataType.INT, np.arange(1000, dtype=np.int32) * 7 + 1, a_ids[::-1].copy()),
                                  b, c, d, x, k, m])
    c_in = ", ".join(str(int(v) * 1_000_003) for v in range(0, 20000, 3))
    k_in = ", ".join(str(int(v)) for v in np.unique(k_raw_sample(seg, 40)))
    for sql in (
            "SELECT d, COUNT(*), SUM(m), MIN(m), MAX(m) FROM t WHERE a IN (8, 15, 29, 701) AND b < 9000 GROUP BY d",
            "SELECT d, COUNT(*), SUM(m) FROM t WHERE a = 22 AND b BETWEEN 300 AND 12000 AND d <> 12 AND x < 0.75 AND k > 200000 GROUP BY d",
            f"SELECT COUNT(*), SUM(m) FROM t WHERE a IN (8, 15) AND c IN ({c_in}) AND b NOT IN (3, 6, 9, 12)",
            f"SELECT COUNT(*), MAX(m) FROM t WHERE a = 71 AND k IN ({k_in})",
            "SELECT d, COUNT(*), SUM(m) FROM t WHERE a = 22 AND b < 9000 GROUP BY d",      # a = 22 is dictId 3: 70 % of the docs are candidates
            "SELECT COUNT(*) FROM t WHERE a = 22 AND b < 3 AND x > 2.0"):
        check_query([seg, seg2], sql, flags_list=ALL_FLAGS, exact_float=True)


def k_raw_sample(seg, count):
    from pinot_b200.segment_writer import DataType as _DT   # noqa: F401
    col = seg.columns["k"]
    vals = np.frombuffer(col.forward_index[col.forward_index.nbytes - 8 * seg.num_docs:].tobytes(), dtype=">i8")
    return vals[:count].astype(np.int64)


FILTERED = ("SELECT SUM(column6) FILTER(WHERE column6 > 5), COUNT(*) FILTER(WHERE column1 IS NOT NULL), "
            "MAX(column3) FILTER(WHERE column3 IS NOT NULL), SUM(column3), AVG(column7) FILTER(WHERE column7 > 0) FROM testTable")
FILTERED_3 = ("SELECT SUM(column6) FILTER(WHERE column6 > 5 OR column6 < 15), COUNT(*) FILTER(WHERE column1 IS NOT NULL), "
              "MAX(column3) FILTER(WHERE column3 IS NOT NULL AND column3 > 0), SUM(column3), "
              "AVG(column7) FILTER(WHERE column7 > 0 AND column7 < 100) FROM testTable")


def test_golden_filtered_aggregations(sv_group):   # InnerSegmentAggregationSingleValueQueriesTest.java:62-93
    seg, g = sv_group
    for sql, exp, st_e in ((FILTERED + " WHERE column3 > 0", (22266008882250, 30000, 2147419555, 32289159189150, 28175373944314, 30000), (150000, 120000, 30000)),
                           (FILTERED, (22266008882250, 30000, 2147419555, 32289159189150, 28175373944314, 30000), (150000, 120000, 30000)),
                           (FILTERED_3, (22266008882250, 30000, 2147419555, 32289159189150, 0, 0), (120000, 90000, 30000))):
        r = native.execute(g, parse_sql(sql))
        row = _row(r.tables[0])
        assert (int(row[0]), row[1], int(row[2]), int(row[3]), int(row[4][0]), row[4][1]) == exp
        st = r.tables[0].stats
        assert (st["num_docs_scanned"], st["num_entries_scanned_post_filter"], st["num_total_docs"]) == st_e
        r.free()


def test_filtered_aggregations_vs_oracle(synth):
    """FILTER(WHERE ...) clauses: keyless and grouped, dense and hash tables, index-backed and raw clause leaves, per segment
    and merged; every group of the main filter exists and functions without a passing doc keep their defaults."""
    segs, g = synth
    d1 = segs[0].columns["c1"].dictionary_values()
    d3 = segs[0].columns["c3"].dictionary_values()
    in4 = ", ".join(str(int(v)) for v in d1[5:9])
    for sql, exact in (
            (f"SELECT d0, d1, SUM(m0) FILTER(WHERE c2 < {int(segs[0].columns['c2'].dictionary_values()[3000])}), COUNT(*) FILTER(WHERE c1 IN ({in4})), "
             f"MIN(m1) FILTER(WHERE c1 IN ({in4})), COUNT(*), AVG(m2) FILTER(WHERE x0 < 0.25 OR c3 = {int(d3[5])}), MAX(m2) FROM t WHERE c1 > {int(d1[100])} GROUP BY d0, d1 LIMIT 100000", True),
            (f"SELECT SUM(m0) FILTER(WHERE x0 < 0.5), COUNT(*) FILTER(WHERE x0 < 0.5), AVG(x1) FILTER(WHERE k0 > 5000000000000), DISTINCTCOUNT(c0) FILTER(WHERE c1 IN ({in4})), "
             f"MAX(m1) FILTER(WHERE c1 < -5) FROM t WHERE c3 <> {int(d3[2])}", False),
            (f"SELECT s0, COUNT(*) FILTER(WHERE t0 BETWEEN 20010 AND 20030), SUM(x0) FILTER(WHERE NOT (c1 IN ({in4}))), DISTINCTCOUNT(d3) FILTER(WHERE x1 > 0.9) FROM t GROUP BY s0 LIMIT 100000", False),
            ("SET numGroupsLimit = 20000000; SELECT k0, COUNT(*) FILTER(WHERE x0 < 0.3), SUM(m0) FILTER(WHERE m0 > 500000) FROM t WHERE x1 < 0.02 GROUP BY k0 LIMIT 100000000", True)):
        check_query(segs, sql, group=g, exact_float=exact)


def test_golden_inter_segment_group_by(sv_group):
    """InterSegmentGroupBySingleValueQueriesTest.java:61-288: the (group -> value) literals of the reference's 4-segment
    group-by results (its ORDER BY / LIMIT are broker-side), from the device-side merge (PB_Q_COMBINE)."""
    from tests.test_oracle_golden import G11_12_SUM1, G11_AVG6, G11_MIN6, G11_SUM1, G12_MIN6, G17_COUNT
    seg, g = sv_group
    C = native.PB_Q_COMBINE
    t = native.execute(g, parse_sql("SELECT column11, SUM(column1), MIN(column6) FROM testTable GROUP BY column11"), C).tables[0].rows()
    assert {k[0]: v[0] for k, v in t.items()} == G11_SUM1 and {k[0]: v[1] for k, v in t.items()} == G11_MIN6
    t = native.execute(g, parse_sql("SELECT column11, column12, SUM(column1) FROM testTable GROUP BY column11, column12"), C).tables[0].rows()
    got = {k: v[0] for k, v in t.items()}
    assert all(got[k] == v for k, v in G11_12_SUM1.items())
    t = native.execute(g, parse_sql("SELECT column12, MIN(column6) FROM testTable GROUP BY column12"), C).tables[0].rows()
    assert {k[0]: v[0] for k, v in t.items()} == G12_MIN6
    t = native.execute(g, parse_sql("SELECT column17, COUNT(*) FROM testTable GROUP BY column17"), C).tables[0].rows()
    got = {k[0]: v[0] for k, v in t.items()}
    assert [(k, got[k]) for k in sorted(got)[:15]] == sorted(G17_COUNT.items())
    t = native.execute(g, parse_sql("SELECT column11, AVG(column6) FROM testTable GROUP BY column11"), C).tables[0].rows()
    assert {k[0]: v[0][0] / v[0][1] for k, v in t.items()} == G11_AVG6


def test_query_from_mmapped_v3_directory(tmp_path):
    """The index buffers handed to pb_segment_stage are views of one mmap'd columns.psf (SingleFileIndexDirectory layout:
    index_map + magic markers): arbitrary byte offsets, read-only, file-backed pages."""
    from pinot_b200.segment_writer import load_v3, write_v3
    native.init()
    seg = datagen.make_segment_synth(4, 70_003, columns=["c1", "c3", "d0", "s0", "t0", "m0", "x0", "k0"])
    back = load_v3(write_v3(seg, str(tmp_path)))
    d1, d3 = seg.columns["c1"].dictionary_values(), seg.columns["c3"].dictionary_values()
    for sql, exact in ((f"SELECT s0, d0, COUNT(*), SUM(m0), MAX(x0) FROM t WHERE c3 IN ({int(d3[2])}, {int(d3[9])}) OR c1 BETWEEN {int(d1[40])} AND {int(d1[90])} GROUP BY s0, d0 LIMIT 100000", False),
                       ("SELECT COUNT(*), MIN(k0), AVG(m0) FROM t WHERE t0 BETWEEN 20003 AND 20011 OR x0 < 0.25", True)):
        check_query([back], sql, exact_float=exact)


def test_var_length_string_dictionary():
    """a .vl; dictionary (VarLengthValueReader.java:41-96) is staged as padded entries: group keys, predicates and
    DISTINCTCOUNT on such a column equal the oracle's"""
    rng = np.random.Generator(np.random.PCG64(11))
    words = [b"a", b"ab", b"abc", b"zebra", b"pinot-b200", b"x" * 37, b"mid", b"", b"q"]
    segs = []
    for i in range(2):
        vals = [words[j] for j in rng.integers(0, len(words) - i, size=20000)]      # the second segment misses a value
        segs.append(make_segment(f"vl{i}", [build_column("s", DataType.STRING, vals, var_length_dictionary=True, inverted=True),
                                            build_column("v", DataType.INT, rng.integers(0, 1000, size=20000))]))
    for sql in ("SELECT s, COUNT(*), SUM(v) FROM t WHERE s > 'ab' AND s <= 'pinot-b200' GROUP BY s LIMIT 100",
                "SELECT COUNT(*), MAX(v) FROM t WHERE s IN ('', 'zebra', 'nosuch') OR s = 'mid'",
                "SET skipIndexes = 's=inverted'; SELECT s, DISTINCTCOUNT(v), MIN(v) FROM t WHERE s != 'q' GROUP BY s LIMIT 100"):
        check_query(segs, sql, flags_list=(0, native.PB_Q_GENERIC_KERNEL))


def test_num_groups_limit_dense_tables_keep_the_first_groups_in_doc_order():
    """numGroupsLimit below the key space: the reference's IntMapBasedHolder creates groups first come first served in doc
    order and drops the rows of later keys (DictionaryBasedGroupKeyGenerator.java:1023-1058).  Per-segment dense tables
    reproduce exactly that set of groups with their full aggregates."""
    segs = [datagen.make_segment_synth(i, 30_000, columns=["c2", "c3", "d1", "d2", "m0", "m1"]) for i in range(2)]
    d2 = segs[0].columns["c2"].dictionary_values()
    for limit in (1, 7, 100, 500, 512, 100000):
        for sql in (f"SET numGroupsLimit = {limit}; SELECT d1, d2, COUNT(*), SUM(m0), MIN(m1) FROM t GROUP BY d1, d2 LIMIT 100000",
                    f"SET numGroupsLimit = {limit}; SELECT c3, d2, COUNT(*), MAX(m0) FROM t WHERE c2 < {int(d2[len(d2) // 3])} GROUP BY c3, d2 LIMIT 100000"):
            q = parse_sql(sql)
            staged = [native.StagedSegment(s) for s in segs]
            g = native.SegmentGroup(staged)
            for flags in (0, native.PB_Q_GENERIC_KERNEL):
                res = native.execute(g, q, flags)
                for i, (t, s) in enumerate(zip(res.tables, segs)):
                    o = oracle.execute(s, q)
                    assert_rows_equal(t.rows(), oracle_rows(o), q, exact_float=True, what=f"limit {limit} segment {i}")
                    assert t.stats["num_groups_limit_reached"] == o.stats["num_groups_limit_reached"], (limit, t.stats, o.stats)
                    assert t.stats["num_docs_scanned"] == o.stats["num_docs_scanned"]
                res.free()
            g.release()


def test_num_groups_limit_hash_tables_never_overflow_or_hang():
    """ADVICE r1 (high): every resident thread used to pass the limit check at once, fill the table and leave absent keys
    probing forever.  Hash tables apply the limit in thread order (documented divergence): at most `limit` groups, the flag
    set, every returned group complete (its aggregates equal the unlimited query's)."""
    segs = [datagen.make_segment_synth(i, 200_000, columns=["k0", "m0", "c2"]) for i in range(2)]
    full_q = parse_sql("SET numGroupsLimit = 10000000; SELECT k0, COUNT(*), SUM(m0) FROM t GROUP BY k0 LIMIT 10000000")
    staged = [native.StagedSegment(s) for s in segs]
    g = native.SegmentGroup(staged)
    full = [oracle_rows(oracle.execute(s, full_q)) for s in segs]
    for limit in (1, 100, 1000, 5000):
        q = parse_sql(f"SET numGroupsLimit = {limit}; SELECT k0, COUNT(*), SUM(m0) FROM t GROUP BY k0 LIMIT 10000000")
        for run in range(3):
            res = native.execute(g, q, 0)
            for i, t in enumerate(res.tables):
                rows = t.rows()
                assert 0 < len(rows) <= limit, (limit, len(rows))
                assert t.stats["num_groups_limit_reached"] == 1
                for k, row in rows.items():
                    assert row == full[i][k], (limit, k, row, full[i][k])      # no partially aggregated group
            res.free()
        res = native.execute(g, q, native.PB_Q_COMBINE)
        rows = res.tables[0].rows()
        assert 0 < len(rows) <= limit and res.tables[0].stats["num_groups_limit_reached"] == 1
        res.free()
    g.release()


def test_distinctcount_on_raw_columns():
    """BaseDistinctAggregateAggregationFunction.java:157-226 (per-group value sets of a no-dictionary column): keyless,
    dense and hash group tables, per segment and merged; sizes and the value sets themselves"""
    rng = np.random.Generator(np.random.PCG64(5))
    segs = []
    for i in range(2):
        n = 40_000 + 1000 * i
        rd = np.round(rng.normal(size=n), 1)
        rd[::101] = -0.0
        segs.append(make_segment(f"rawdc{i}", [
            build_column("g", DataType.INT, rng.integers(0, 12, size=n)), build_column("h", DataType.INT, rng.integers(0, 5, size=n)),
            build_column("ri", DataType.INT, rng.integers(-50, 50, size=n), dictionary=False),
            build_column("rl", DataType.LONG, rng.integers(-10**12, 10**12, size=n) // 10**11 * 10**11, dictionary=False),
            build_column("rd", DataType.DOUBLE, rd, dictionary=False),
            build_column("k", DataType.LONG, rng.integers(0, 3000, size=n), dictionary=False),
            build_column("f", DataType.INT, rng.integers(0, 100, size=n))]))
    for sql in ("SELECT DISTINCTCOUNT(ri), DISTINCTCOUNT(rl), DISTINCTCOUNT(rd), COUNT(*) FROM t WHERE f < 60",
                "SELECT g, h, DISTINCTCOUNT(ri), DISTINCTCOUNT(rd), DISTINCTCOUNT(f), SUM(f) FROM t WHERE f >= 10 GROUP BY g, h LIMIT 1000",
                "SELECT k, DISTINCTCOUNT(ri), COUNT(*) FROM t GROUP BY k LIMIT 100000"):
        check_query(segs, sql)


def _expected_trim(rows, q, combined):
    """what TableResizer keeps: the trim_size best groups by the first ORDER BY expression (+ every tie with the last)"""
    size, thr = q.trim(combined)
    if not size or len(rows) <= thr or len(rows) <= size:
        return rows
    kind, idx, desc = q.order_by[0]

    def key(item):
        k, row = item
        v = k[idx] if kind == 0 else row[idx]
        if isinstance(v, tuple):          # AVG: (sum, count); no input: AvgAggregationFunction's DEFAULT_FINAL_RESULT
            v = v[0] / v[1] if v[1] else float("-inf")
        return v
    vals = sorted((key(it) for it in rows.items()), reverse=desc)
    cut = vals[size - 1]
    return {k: r for k, r in rows.items() if (key((k, r)) >= cut if desc else key((k, r)) <= cut)}


def test_order_by_limit_trim_on_the_device():
    """ORDER BY ... LIMIT: the server-side trim of the combine layer (GroupByUtils.getTableCapacity = max(5 x LIMIT,
    minServerGroupTrimSize) groups once the table passes groupTrimThreshold; TableResizer) done at hand-back: the kept groups
    are exactly the best ones by the first ORDER BY expression (ties with the last kept group included), values untouched."""
    segs = [datagen.make_segment_synth(i, 60_000, columns=["c2", "c3", "d1", "d2", "m0", "m1", "k0"]) for i in range(2)]
    staged = [native.StagedSegment(s) for s in segs]
    g = native.SegmentGroup(staged)
    opts = "SET groupTrimThreshold = 100; SET minServerGroupTrimSize = 20; SET minSegmentGroupTrimSize = 30; "
    for tail in ("ORDER BY SUM(m0) DESC LIMIT 3", "ORDER BY SUM(m0) ASC LIMIT 3", "ORDER BY COUNT(*) DESC LIMIT 2", "ORDER BY MIN(m1) ASC LIMIT 1",
                 "ORDER BY MAX(m1) DESC, d2 LIMIT 4", "ORDER BY AVG(m0) DESC LIMIT 3", "ORDER BY d2 DESC, c3 ASC LIMIT 2", "ORDER BY c3 LIMIT 1"):
        sql = opts + "SELECT c3, d2, SUM(m0), COUNT(*), MIN(m1), MAX(m1), AVG(m0) FROM t WHERE c2 >= 0 GROUP BY c3, d2 " + tail
        q = parse_sql(sql)
        orc = [oracle.execute(s, q) for s in segs]
        for run in range(3):                       # also through the plan cache / graph replay
            res = native.execute(g, q, native.PB_Q_COMBINE)
            exp = _expected_trim(combined_rows(oracle.combine(orc), q), q, True)
            assert 20 <= len(exp) < 2048
            assert_rows_equal(res.tables[0].rows(), exp, q, exact_float=True, what=f"combined trim: {tail}")
            res.free()
        res = native.execute(g, q, 0)
        for i, (t, o) in enumerate(zip(res.tables, orc)):
            assert_rows_equal(t.rows(), _expected_trim(oracle_rows(o), q, False), q, exact_float=True, what=f"segment {i} trim: {tail}")
        res.free()
    # a hash table (raw LONG key) ordered by its key and by an aggregate; and no trim below the threshold
    for tail in ("ORDER BY k0 DESC LIMIT 3", "ORDER BY SUM(m0) DESC LIMIT 2"):
        q = parse_sql("SET numGroupsLimit = 10000000; " + opts + "SELECT k0, SUM(m0), COUNT(*) FROM t GROUP BY k0 " + tail)
        orc = [oracle.execute(s, q) for s in segs]
        res = native.execute(g, q, native.PB_Q_COMBINE)
        exp = _expected_trim(combined_rows(oracle.combine(orc), q), q, True)
        assert_rows_equal(res.tables[0].rows(), exp, q, exact_float=True, what=f"hash trim: {tail}")
        res.free()
    q = parse_sql("SELECT d1, SUM(m0) FROM t GROUP BY d1 ORDER BY SUM(m0) DESC LIMIT 3")      # 16 groups: far below any threshold
    res = native.execute(g, q, native.PB_Q_COMBINE)
    assert len(res.tables[0].rows()) == 16
    res.free()
    g.release()


@pytest.mark.parametrize("compression", ["LZ4", "LZ4_LENGTH_PREFIXED", "SNAPPY"])
def test_chunk_compressed_raw_columns(compression):
    """Raw forward indexes written with a chunk codec (ChunkCompressionType LZ4 / LZ4_LENGTH_PREFIXED / SNAPPY, offsets as ints
    (v2) or longs (v4), short last chunk): the compressed bytes are staged and decoded on the device (pb_chunk_decode_kernel);
    predicates, group keys, aggregation inputs and DISTINCTCOUNT value sets read from the decoded value area."""
    native.init()
    rng = np.random.default_rng(77)
    segs = []
    for si, (n, version, per_chunk) in enumerate(((30_123, 2, 1000), (18_001, 4, 4096))):
        d = rng.integers(0, 9, n).astype(np.int32)
        k = np.cumsum(rng.integers(-2, 6, n)).astype(np.int64) - 20_000            # compresses into long matches
        i = rng.integers(-50, 50, n).astype(np.int32)
        x = np.round(rng.normal(0, 5, n), 1)                                      # few distinct doubles
        f = rng.integers(0, 1000, n).astype(np.float32) / 8
        r = rng.integers(-2**62, 2**62, n).astype(np.int64)                       # incompressible: literal-only chunks
        raw = dict(dictionary=False, raw_compression=compression, raw_version=version, raw_docs_per_chunk=per_chunk)
        segs.append(make_segment(f"z{si}", [build_column("d", DataType.INT, d), build_column("k", DataType.LONG, k, **raw),
                                            build_column("i", DataType.INT, i, **raw), build_column("x", DataType.DOUBLE, x, **raw),
                                            build_column("f", DataType.FLOAT, f, **raw), build_column("r", DataType.LONG, r, **raw)]))
    check_query(segs, "SELECT d, COUNT(*), SUM(k), MIN(x), MAX(f), AVG(i) FROM t WHERE k > -15000 AND x < 4.5 AND i <> 7 GROUP BY d LIMIT 100")
    check_query(segs, "SELECT i, COUNT(*), MAX(r), DISTINCTCOUNT(f) FROM t WHERE f BETWEEN 10 AND 90 GROUP BY i LIMIT 1000")
    check_query(segs, "SELECT COUNT(*), MIN(r), MAX(r), SUM(x) FROM t WHERE r > 0", exact_float=False)


def test_malformed_compressed_chunk_is_rejected():
    native.init()
    rng = np.random.default_rng(3)
    n = 5000
    k = np.cumsum(rng.integers(0, 3, n)).astype(np.int64)
    col = build_column("k", DataType.LONG, k, dictionary=False, raw_compression="LZ4")
    fwd = col.forward_index
    off1 = int.from_bytes(fwd[28 + 4:28 + 8].tobytes(), "big")
    fwd[off1] = 0x0F                                     # chunk 1 now opens with "no literals, match" before any output exists
    fwd[off1 + 1:off1 + 3] = (9, 0)
    seg = make_segment("bad", [build_column("d", DataType.INT, rng.integers(0, 4, n).astype(np.int32)), col])
    staged = native.StagedSegment(seg)
    group = native.SegmentGroup([staged])
    with pytest.raises(native.PinotB200Error) as e:
        native.execute(group, parse_sql("SELECT d, SUM(k) FROM t GROUP BY d LIMIT 10"), 0)
    assert "do not decode" in str(e.value)


def test_predicates_on_several_wide_raw_columns():
    """Three scan leaves over raw LONG / DOUBLE / INT columns (160 bits per row) do not fit the per-warp stages of shared
    memory: the most selective one is streamed, the others run on its survivors (DevLeaf::gather) whatever the selectivity."""
    native.init()
    rng = np.random.default_rng(12)
    n = 40_007
    cols = [build_column("d", DataType.INT, rng.integers(0, 5, n).astype(np.int32)),
            build_column("k", DataType.LONG, rng.integers(-10**12, 10**12, n).astype(np.int64), dictionary=False),
            build_column("x", DataType.DOUBLE, rng.normal(0, 5, n), dictionary=False),
            build_column("y", DataType.DOUBLE, rng.normal(0, 5, n), dictionary=False),
            build_column("i", DataType.INT, rng.integers(-50, 50, n).astype(np.int32), dictionary=False)]
    segs = [make_segment("wide", cols)]
    check_query(segs, "SELECT d, COUNT(*), SUM(i), MIN(x) FROM t WHERE k > -900000000000 AND x < 6.5 AND y > -7 AND i <> 7 GROUP BY d LIMIT 100")
    check_query(segs, "SELECT COUNT(*), MAX(k) FROM t WHERE k > 0 AND x < 0 AND y > 0")


def test_is_null_predicates_over_null_value_vectors():
    """IS NULL / IS NOT NULL = BitmapBasedFilterOperator over the column's null-value vector (FilterPlanNode.java:294-307;
    the counts of SegmentWithNullValueVectorTest :242-273 on generated data), combined with scan leaves, OR and NOT."""
    from tests.test_cpu_formats import _null_segment
    native.init()
    seg, d, i, k, i_null, k_null = _null_segment(60_000, seed=8)
    segs = [seg]
    for sql in ("SELECT COUNT(*) FROM t WHERE i IS NOT NULL", "SELECT COUNT(*) FROM t WHERE i IS NULL",
                "SELECT COUNT(*) FROM t WHERE i IS NOT NULL AND k > 500000", "SELECT COUNT(*), SUM(k) FROM t WHERE i IS NULL OR k IS NULL",
                "SELECT d, COUNT(*), MAX(k) FROM t WHERE NOT (i IS NULL) AND k IS NULL AND d < 3 GROUP BY d LIMIT 10",
                "SELECT COUNT(*) FROM t WHERE z IS NULL", "SELECT d, COUNT(*) FROM t WHERE z IS NOT NULL AND i IS NULL GROUP BY d LIMIT 10"):
        check_query(segs, sql)
    res = native.execute(native.SegmentGroup([native.StagedSegment(seg)]), parse_sql("SELECT COUNT(*) FROM t WHERE i IS NULL"), 0)
    assert res.tables[0].rows()[()][0] == int(i_null.sum())
    res.free()
