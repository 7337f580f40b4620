"""The plan cache (-m gpu): pb_result_free parks a result whose plan is reusable in its segment group; the next identical
query replays it -- eagerly the first time, then as one CUDA graph launch.  Every run must still equal the oracle: the
query's work is redone each time, only the planning is reused."""
import threading

import numpy as np
import pytest

from oracle import oracle
from pinot_b200 import datagen, native
from pinot_b200.query import parse_sql
from tests.parity import assert_rows_equal, combined_rows, oracle_rows

pytestmark = pytest.mark.gpu
COLS = ["c1", "c2", "c3", "d0", "d1", "d2", "m0", "m1", "m2", "x0", "k0"]


@pytest.fixture(scope="module")
def table():
    native.init()
    segs = [datagen.make_segment_synth(i, 80_000 + 3000 * i, columns=COLS, vary_dim_dictionaries=(i == 1)) for i in range(3)]
    staged = [native.StagedSegment(s) for s in segs]
    group = native.SegmentGroup(staged)
    yield segs, group
    group.release()
    for s in staged:
        s.release()


def _queries(segs):
    d2 = segs[0].columns["c2"].dictionary_values()
    d3 = segs[0].columns["c3"].dictionary_values()
    k2, k3 = int(d2[len(d2) // 2]), int(d3[len(d3) // 3])
    return [
        datagen.config2_sql(segs, 16),                                                        # selective: row-group aggregation
        datagen.config2_sql(segs, 500),                                                       # 25 %: row-group aggregation
        f"SELECT COUNT(*), SUM(m0), MIN(m1), MAX(m2) FROM t WHERE c2 < {k2}",                 # keyless
        f"SELECT d0, DISTINCTCOUNT(c3), SUM(m1) FROM t WHERE c2 < {k2} GROUP BY d0 LIMIT 100000",
        f"SELECT d1, SUM(m0) FILTER(WHERE c3 < {k3}), COUNT(*) FILTER(WHERE c3 < {k3}), COUNT(*) FROM t WHERE c2 < {k2} GROUP BY d1 LIMIT 100000",
        "SET numGroupsLimit = 10000000; SELECT k0, SUM(m0), COUNT(*) FROM t WHERE c3 > %d GROUP BY k0 LIMIT 10000000" % k3,   # hash table
        f"SELECT d2, COUNT(*), SUM(x0) FROM t WHERE c1 IN ({int(segs[0].columns['c1'].dictionary_values()[5])}) OR c3 = {k3} GROUP BY d2 LIMIT 100000",   # inverted-index leaves
        "SELECT d2, COUNT(*), SUM(m2) FROM t GROUP BY d2 LIMIT 100000",                       # match all
    ]


def test_replays_equal_the_oracle(table):
    segs, group = table
    for sql in _queries(segs):
        q = parse_sql(sql)
        orc = [oracle.execute(s, q) for s in segs]
        exp_c = combined_rows(oracle.combine(orc), q)
        for flags, what in ((native.PB_Q_COMBINE, "combined"), (0, "per segment")):
            for run in range(5):       # build, eager replay, graph capture + launch, graph launch, graph launch
                r = native.execute(group, q, flags)
                if flags:
                    assert_rows_equal(r.tables[0].rows(), exp_c, q, exact_float="x0" not in sql, what=f"{what} run {run}: {sql[:60]}")
                    assert r.tables[0].stats["num_docs_scanned"] == sum(o.stats["num_docs_scanned"] for o in orc)
                else:
                    for i, (t, o) in enumerate(zip(r.tables, orc)):
                        assert_rows_equal(t.rows(), oracle_rows(o), q, exact_float="x0" not in sql, what=f"{what} run {run} seg {i}: {sql[:60]}")
                        for key in ("num_docs_scanned", "num_entries_scanned_post_filter", "num_total_docs"):
                            assert t.stats[key] == o.stats[key]
                r.free()


def test_a_live_result_is_never_replayed_under_its_holder(table):
    segs, group = table
    q = parse_sql(datagen.config2_sql(segs, 16))
    exp = combined_rows(oracle.combine([oracle.execute(s, q) for s in segs]), q)
    held = [native.execute(group, q, native.PB_Q_COMBINE) for _ in range(3)]        # three results alive at once
    assert len({h._rh.value for h in held}) == 3
    snapshots = [{k: list(v) for k, v in h.tables[0].rows().items()} for h in held]
    for h in held:
        h.free()
    again = [native.execute(group, q, native.PB_Q_COMBINE) for _ in range(3)]       # takes the three parked plans back
    for r, snap in zip(again, snapshots):
        assert_rows_equal(r.tables[0].rows(), exp, q, exact_float=True, what="replayed")
        assert {k: list(v) for k, v in r.tables[0].rows().items()} == snap
        r.free()


def test_interleaved_queries_and_threads(table):
    """BaseCombineOperator.java:100-141 calls nextBlock() for different segments from the pool's worker threads at the
    same time: concurrent callers on one-segment groups (and on the shared group), each through its own stream."""
    segs, group = table
    sqls = _queries(segs)[:5]
    qs = [parse_sql(s) for s in sqls]
    exps = [[oracle_rows(oracle.execute(s, q)) for s in segs] for q in qs]
    single = [native.SegmentGroup([native.StagedSegment(s)]) for s in segs]
    errors = []

    def worker(tid):
        try:
            for it in range(6):
                qi = (tid + it) % len(qs)
                si = (tid * 7 + it) % len(segs)
                r = native.execute(single[si], qs[qi], 0)
                assert_rows_equal(r.tables[0].rows(), exps[qi][si], qs[qi], exact_float=True, what=f"thread {tid} it {it}")
                r.free()
        except Exception as e:      # pragma: no cover
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[:3]
    for g in single:
        g.release()
