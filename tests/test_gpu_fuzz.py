"""Seeded differential fuzz of the device against the exact reference (tests/reference.py) and the oracle, over tables and
queries built to reach every kernel path the planner can choose (tests/fuzz_gen.py), plus two deterministic cases for the
exact-integer sums of the CTA-private table.

Every call's plan (native.Result.plan_info) is appended to the JSON-lines file named by PB_FUZZ_PLAN_LOG, if set:
tests/test_gpu_kernel_paths.py runs this module in child processes under each tuning knob and checks from those logs that
every kernel path was reached.  PB_FUZZ_SEEDS="1,2" narrows the seeds, PB_FUZZ_MAX_DOCS caps the docs per seed."""
import json
import os

import numpy as np
import pytest

from oracle import oracle
from pinot_b200 import native
from pinot_b200.query import AggOp, parse_sql
from pinot_b200.segment_writer import DataType, build_column, build_dict_column, make_segment
from tests import fuzz_gen
from tests.parity import assert_rows_equal, combined_rows, oracle_rows
from tests.reference import Col, assert_matches_reference, concat, keyless_nan_minmax, reference, without_aggregations

SEEDS = [int(s) for s in os.environ["PB_FUZZ_SEEDS"].split(",")] if os.environ.get("PB_FUZZ_SEEDS") else list(range(8))
QUERIES_PER_SEED = 6
MAX_DOCS = int(os.environ.get("PB_FUZZ_MAX_DOCS", "600000"))       # docs per seed
FLAGS = (0, native.PB_Q_GENERIC_KERNEL, native.PB_Q_NO_TMA)


@pytest.fixture(scope="module", autouse=True)
def _device():
    native.init()


def _log_plan(res, n_segs, what):
    path = os.environ.get("PB_FUZZ_PLAN_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"what": what, "n_segs": n_segs, **res.plan_info}) + "\n")


def _vs_oracle(got, exp, q, skip, what):
    g2, e2, q2 = without_aggregations(got, exp, q, skip)
    assert_rows_equal(g2, e2, q2, exact_float=False, what=what, sums=False)


def run_and_check(group, segs, srcs, sql, what, per_segment=True, replays=0):
    q = parse_sql(sql)
    orc = [oracle.execute(s, q) for s in segs]
    skip = keyless_nan_minmax(q, srcs)
    ref_all = reference(concat(srcs), q)
    ref_seg = [reference(s, q) for s in srcs] if per_segment else None
    for flags in FLAGS:
        if per_segment:
            res = native.execute(group, q, flags)
            _log_plan(res, len(segs), what)
            for i, (t, o) in enumerate(zip(res.tables, orc)):
                w = f"{what} flags={flags} segment {i}: {sql}"
                assert_matches_reference(t.rows(), ref_seg[i], q, w)
                _vs_oracle(t.rows(), oracle_rows(o), q, skip, w)
                for key in ("num_docs_scanned", "num_entries_scanned_post_filter", "num_total_docs"):
                    assert t.stats[key] == o.stats[key], f"{w}: {key}: {t.stats[key]} != {o.stats[key]}"
            res.free()
        exp = combined_rows(oracle.combine(orc), q)
        for rep in range(1 + (replays if flags == 0 else 0)):      # rep 1: plan-cache replay, rep 2: its CUDA graph
            res = native.execute(group, q, flags | native.PB_Q_COMBINE)
            _log_plan(res, len(segs), what)
            t = res.tables[0]
            w = f"{what} flags={flags} combined (run {rep}): {sql}"
            assert_matches_reference(t.rows(), ref_all, q, w)
            _vs_oracle(t.rows(), exp, q, skip, w)
            assert t.stats["num_docs_scanned"] == sum(o.stats["num_docs_scanned"] for o in orc), w
            assert t.stats["num_total_docs"] == sum(s.num_docs for s in segs), w
            res.free()


def _group(segs):
    staged = [native.StagedSegment(s) for s in segs]
    return staged, native.SegmentGroup(staged)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_fuzz_against_reference(seed):
    segs, srcs, facts = fuzz_gen.make_tables(seed, MAX_DOCS)
    staged, g = _group(segs)
    rng = np.random.default_rng(seed)
    try:
        for qi in range(QUERIES_PER_SEED):
            sql = fuzz_gen.make_query(rng, srcs[0])
            # per-segment dense tables of 2^24 slots for many segments would take gigabytes: merged only
            per_seg = not ("kwa" in sql.split("GROUP BY")[-1] and len(segs) > 3)
            run_and_check(g, segs, srcs, sql, f"seed {seed} query {qi}", per_segment=per_seg, replays=2 if qi == 0 else 0)
    finally:
        g.release()
        for s in staged:
            s.release()


@pytest.mark.gpu
def test_rows_kernel_with_8_byte_fields_over_many_segments():
    """pb_agg_rows_kernel at RW = 8 over 20 segments (more than 16: its descriptors then come from global memory): LONG and
    DOUBLE value fields of 8 bytes, a FLOAT field, IEEE edge values in MIN.  The filter keeps 40 % of every segment, so
    every segment reads a row group."""
    segs, srcs = [], []
    for si in range(20):
        nd = (1023, 1025, 2049, 4097)[si % 4]
        r = np.random.default_rng(300 + si)
        cols, src = [], {}
        for name, dt, d in (("k", DataType.INT, np.array([-5, 0, 7])), ("f", DataType.INT, np.arange(10)),
                            ("vl", DataType.LONG, np.array([-(2 ** 62), -3, 0, 11, 2 ** 61])),
                            ("ve", DataType.DOUBLE, fuzz_gen.EDGE_DOUBLES), ("vd", DataType.DOUBLE, np.array([-1e15, -0.5, 1.0, 3e15])),
                            ("vf", DataType.FLOAT, np.array([-2.5, 0.125, 7.0], dtype=np.float32))):
            ids = r.integers(0, len(d), nd)
            cols.append(fuzz_gen._dict_col(name, dt, d, ids))
            src[name] = fuzz_gen._src(dt, d, ids)
        segs.append(make_segment(f"rows{si}", cols))
        srcs.append(src)
    staged, g = _group(segs)
    try:
        sql = "SELECT k, SUM(vl), MIN(ve), MAX(ve), MAX(vd), AVG(vf), COUNT(*) FROM t WHERE f < 4 GROUP BY k LIMIT 100"
        run_and_check(g, segs, srcs, sql, "rows RW=8", replays=2)
        res = native.execute(g, parse_sql(sql), native.PB_Q_COMBINE)
        if _expect_rows_kernel():
            assert res.plan_info["agg_kernel"] == 3 and res.plan_info["rows_rw"] == 8, res.plan_info
        res.free()
    finally:
        g.release()
        for s in staged:
            s.release()


# ---- deterministic: the exact-integer sums of the CTA-private table ----

def _carry_table(n_docs, seed=5):
    """one dense group per key, INT inputs alternating about 2^31 - 1 and about -2^31, LONG inputs about +-2^40: every
    CTA replica's low half wraps again and again.  A filter keeps half the docs, so the call reads row groups.  neg / pos /
    nan: MIN / MAX inputs of one sign or all NaN, whose results depend on how the CTA table's cells start."""
    r = np.random.default_rng(seed)
    k = r.integers(0, 4, n_docs)
    alt = np.arange(n_docs) % 2 == 0
    vi = np.where(alt, 2 ** 31 - 1 - r.integers(0, 8, n_docs), -(2 ** 31) + r.integers(0, 8, n_docs)).astype(np.int64)
    vl = np.where(alt, 2 ** 40 - r.integers(0, 8, n_docs), -(2 ** 40) + r.integers(0, 3, n_docs)).astype(np.int64)
    f = r.integers(0, 2, n_docs)
    cols = [build_column("k", DataType.INT, k.astype(np.int32)), build_column("vi", DataType.INT, vi.astype(np.int32)),
            build_column("vl", DataType.LONG, vl), build_column("f", DataType.INT, f.astype(np.int32))]
    src = {"k": Col(k, DataType.INT), "vi": Col(vi, DataType.INT), "vl": Col(vl, DataType.LONG), "f": Col(f, DataType.INT)}
    for name, dt, d in (("neg", DataType.DOUBLE, fuzz_gen.NEG_DOUBLES), ("pos", DataType.INT, np.array([3, 17, 2 ** 30])),
                        ("nan", DataType.FLOAT, np.array([np.nan], dtype=np.float32))):     # (4 bytes: the LONG row still fits 256 bits)
        ids = r.integers(0, len(d), n_docs)
        cols.append(fuzz_gen._dict_col(name, dt, d, ids))
        src[name] = fuzz_gen._src(dt, d, ids)
    return make_segment("carry", cols), src


def _smem_on():
    return os.environ.get("PB_AGG_SMEM", "1") != "0"


def _expect_rows_kernel():
    return os.environ.get("PB_AGG_ROWS", "1") != "0" and os.environ.get("PB_ROW_GROUPS", "1") != "0"


def _expect_exact():
    return _expect_rows_kernel() and _smem_on() and os.environ.get("PB_AGG_EXACT_INT", "1") != "0"


@pytest.mark.gpu
def test_exact_integer_sum_carries():
    """INT: 2 M docs x 2^31 < 2^53 -- exact mode, sums must equal the integer sums exactly.  LONG: 8000 docs x 2^40 < 2^53.
    Both calls update the CTA-private table (enough matches per slot); the second query of each is pb_agg_smem_kernel (a
    FILTER clause rules out the rows kernel), with a clause that leaves its functions no input."""
    extremes = "MAX(neg), MIN(pos), MIN(nan), MAX(nan)"
    for n_docs, cols in ((2_000_000, "SUM(vi), AVG(vi), MIN(vi), MAX(vi)"), (8_000, "SUM(vl), AVG(vl), SUM(vi)")):
        seg, src = _carry_table(n_docs)
        staged, g = _group([seg])
        try:
            sql = f"SELECT k, COUNT(*), {cols}, {extremes} FROM t WHERE f = 0 GROUP BY k LIMIT 100"
            run_and_check(g, [seg], [src], sql, f"carry {n_docs}", replays=2)
            q = parse_sql(sql)
            res = native.execute(g, q, native.PB_Q_COMBINE)
            pi = res.plan_info
            sums = sum(1 << a for a, agg in enumerate(q.aggregations) if agg.op in (AggOp.SUM, AggOp.AVG))
            if _expect_rows_kernel():
                assert pi["agg_kernel"] == 3 and (pi["st_replicas"] > 0) == _smem_on(), pi
            assert pi["exact_int_mask"] == (sums if _expect_exact() else 0), pi
            res.free()
            sql = f"SELECT k, {extremes}, MAX(vi) FILTER(WHERE f = 1), MIN(neg) FILTER(WHERE f = 1), COUNT(*) FILTER(WHERE f = 1) " \
                  f"FROM t WHERE f = 0 GROUP BY k LIMIT 100"
            run_and_check(g, [seg], [src], sql, f"carry {n_docs} FILTER")
            res = native.execute(g, parse_sql(sql), native.PB_Q_COMBINE)
            assert res.plan_info["agg_kernel"] == 2 or not _smem_on(), res.plan_info
            res.free()
        finally:
            g.release()
            staged[0].release()


@pytest.mark.gpu
def test_cta_table_at_the_shared_memory_budget():
    """One SUM over 17066 dense slots is exactly 200 KB of CTA table (4-byte row counts + 8-byte sums): one replica.
    17067 slots is one slot past the budget: no CTA table.  Under PB_AGG_SMEM_MIN=0 the one replica is also used."""
    n = 60_000
    r = np.random.default_rng(11)
    f = r.integers(0, 2, n)
    v = r.integers(-1000, 1000, n)
    cols = [build_column("f", DataType.INT, f.astype(np.int32)), build_column("v", DataType.INT, v.astype(np.int32))]
    src = {"f": Col(f, DataType.INT), "v": Col(v, DataType.INT)}
    for name, card in (("kin", 17_066), ("kout", 17_067)):
        d = np.arange(card, dtype=np.int64) * 5
        ids = r.integers(0, card, n)
        cols.append(fuzz_gen._dict_col(name, DataType.INT, d, ids))
        src[name] = fuzz_gen._src(DataType.INT, d, ids)
    seg = make_segment("budget", cols)
    staged, g = _group([seg])
    try:
        for key, replicas in (("kin", 1), ("kout", 0)):
            sql = f"SELECT {key}, SUM(v) FROM t WHERE f = 0 GROUP BY {key} LIMIT 100000"
            run_and_check(g, [seg], [src], sql, f"budget {key}")
            res = native.execute(g, parse_sql(sql), native.PB_Q_COMBINE)
            assert res.plan_info["st_replicas"] == (replicas if _smem_on() else 0), (key, res.plan_info)
            res.free()
    finally:
        g.release()
        staged[0].release()


@pytest.mark.gpu
def test_dictionary_widths_up_to_24_bits():
    """Streamed dictIds of 17, 20 (specialised filter kernels) and 24 bits (general kernel only): single leaves, a set, a
    conjunction, and the general kernel for all of them (PB_Q_GENERIC_KERNEL in run_and_check)"""
    segs, srcs = [], []
    for si, n in enumerate((40_000, 33_000)):
        r = np.random.default_rng(500 + si)
        cols, src = [], {}
        for name, dt, d in (("k", DataType.INT, np.array([-5, 0, 7])), ("w17", DataType.INT, np.arange(2 ** 16 + 1) * 3),
                            ("w20", DataType.LONG, np.arange(2 ** 19 + 1) - 7), ("w24", DataType.INT, np.arange(2 ** 23 + 1))):
            ids = r.integers(0, len(d), n)
            ids[:2] = [len(d) - 1, 0]                  # the last entry occurs, the column is not sorted
            cols.append(fuzz_gen._dict_col(name, dt, d.astype(np.int64), ids))
            src[name] = fuzz_gen._src(dt, d.astype(np.int64), ids)
        segs.append(make_segment(f"wide{si}", cols))
        srcs.append(src)
    staged, g = _group(segs)
    try:
        for where in ("w17 < 30000", "w20 >= 400000", "w24 < 4194304", "w24 IN (0, 5, 8388608, 77)",
                      "w20 BETWEEN 1000 AND 90000 AND w24 > 100 AND w17 <> 9"):
            run_and_check(g, segs, srcs, f"SELECT k, COUNT(*), SUM(w24), MAX(w20) FROM t WHERE {where} GROUP BY k LIMIT 10", f"widths {where}")
    finally:
        g.release()
        for s in staged:
            s.release()


@pytest.mark.gpu
def test_exact_integer_mode_edge():
    """plan_rows_kernel turns the exact-integer mode on when bound < 2^53 and docs_all < 2^53 / bound (integer division;
    bound = the larger |first|, |last| dictionary entry, docs_all = every doc of the call).  One LONG column just inside,
    one just outside: the mask flips exactly there, and both results match the reference."""
    n = [6_000, 14_000]
    docs_all = sum(n)
    b_in = (2 ** 53) // (docs_all + 1)              # 2^53 // b_in >= docs_all + 1 > docs_all: exact
    b_out = (2 ** 53) // docs_all + 1                # 2^53 // b_out < docs_all: double
    assert docs_all < (2 ** 53) // b_in and not docs_all < (2 ** 53) // b_out
    segs, srcs = [], []
    for si, nd in enumerate(n):
        r = np.random.default_rng(90 + si)
        k, f = r.integers(0, 3, nd), r.integers(0, 2, nd)
        cols, src = [build_column("k", DataType.INT, k.astype(np.int32)), build_column("f", DataType.INT, f.astype(np.int32))], \
            {"k": Col(k, DataType.INT), "f": Col(f, DataType.INT)}
        for name, b in (("lin", b_in), ("lout", b_out)):
            d = np.array([-b, -3, 5, b], dtype=np.int64)
            ids = r.integers(0, 4, nd)
            cols.append(build_dict_column(name, DataType.LONG, d, ids.astype(np.uint32)))
            src[name] = Col(d[ids], DataType.LONG)
        segs.append(make_segment(f"edge{si}", cols))
        srcs.append(src)
    staged, g = _group(segs)
    try:
        for col, exact in (("lin", True), ("lout", False)):
            sql = f"SELECT k, SUM({col}), AVG({col}) FROM t WHERE f = 1 GROUP BY k LIMIT 10"
            run_and_check(g, segs, srcs, sql, f"mode edge {col}")
            res = native.execute(g, parse_sql(sql), native.PB_Q_COMBINE)
            pi = res.plan_info
            assert pi["exact_int_mask"] == (0b11 if exact and _expect_exact() else 0), (col, pi)
            res.free()
    finally:
        g.release()
        for s in staged:
            s.release()
