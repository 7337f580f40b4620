"""The all-to-all merge of hash group tables across ranks, held to the exact reference on ONE GPU by exchanging the partitions
of simulated ranks.

The ranks are those of tests/test_gpu_rank_merge.py (Ranks / simulate_ranks: one segment group per rank on device 0, the
global dictionaries agreed, every rank's query run with PB_Q_COMBINE | PB_Q_DEFER_FINALIZE).  Every rank then partitions its
hash table for n ranks (pb_result_hash_partition: the real pb_hash_count_kernel and pb_hash_pack_kernel), and torch copies of
the packed tuples build each destination's receive buffer from the sources' slices, in source-rank order, with the counter
cells of all ranks rank-major and their layout words: what comm_merge_hash's grouped ncclSend / ncclRecv and all-gathers
deliver.  pb_result_hash_merge_received (the real pb_hash_merge_kernel into a table sized for what arrived) and
pb_result_finalize then hand back each rank's partition, and the union of the partitions is judged by tests/reference.py over
all segments of all ranks.  NCCL itself is not covered here (tests/multi_gpu_worker.py runs it where two GPUs exist).

PB_FUZZ_SEEDS="1,3" narrows the fuzz seeds."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from pinot_b200 import native
from pinot_b200.segment_writer import DataType, build_column, make_segment, with_nulls
from tests import fuzz_gen
from tests.parity import assert_rows_equal, combined_rows
from tests.reference import Col, SumRef, assert_matches_reference
from tests.test_cpu_null_handling import INT_NULL, NH
from tests.test_gpu_rank_merge import (HASH, PB_ERR_STATE, PB_ERR_UNSUPPORTED, _bits, _raises, _same_except_float_sums, device_view,
                                       simulate_ranks)

pytestmark = pytest.mark.gpu

# seed 1: 24 segments (8 ranks hold three each); seed 3: 5 segments, contiguous shards leave one rank a single 31-doc
# segment; seed 2: 4097 values in kwb (kwa, kwb is a hash table)
SEEDS = [int(s) for s in os.environ["PB_FUZZ_SEEDS"].split(",")] if os.environ.get("PB_FUZZ_SEEDS") else [1, 2, 3]
QUERIES_PER_SEED = 4
MAX_DOCS = 200_000
UNLIMITED = "SET numGroupsLimit = 100000000; "
REACHED = []                    # one record per rank of every exchange: what, n_ranks, rank, key_words, tuples received


@pytest.fixture(scope="module", autouse=True)
def _device():
    native.init()
    yield
    torch.cuda.empty_cache()


# ---- the exchange ----

def exchange(ranks, order=None):
    """Every rank partitions for n ranks; each destination receives the sources' slices for it concatenated in source order
    (`order`, default rank order), the counter cells of all ranks rank-major and the layout words of all ranks.  Returns
    the receive buffers (kept alive until the merges have run) and their tuple counts."""
    n = ranks.n
    parts = [res.hash_partition(n) for res in ranks.results]
    for res in ranks.results:
        res.wait()
    layouts = [p[5] for p in parts]
    cells = torch.cat([device_view(p[3], 8 * p[4]) for p in parts])          # (a copy: every merge rewrites its own cells)
    received = []
    for dst in range(n):
        chunks, n_tuples = [], 0
        for src in (order or range(n)):
            ptr, counts, words = parts[src][0], parts[src][1], parts[src][2]
            if counts[dst]:
                chunks.append(device_view(ptr + 8 * words * sum(counts[:dst]), 8 * words * counts[dst]))
                n_tuples += counts[dst]
        received.append((torch.cat(chunks) if chunks else torch.empty(8, dtype=torch.uint8, device="cuda"), n_tuples))
    torch.cuda.synchronize()
    return received, cells, layouts


def merged_partitions(ranks, order=None):
    """exchange, merge what each rank received, finalize: every rank's table"""
    received, cells, layouts = exchange(ranks, order)
    for rank, (res, (buf, n_tuples)) in enumerate(zip(ranks.results, received)):
        res.hash_merge_received(buf.data_ptr(), n_tuples, cells.data_ptr(), layouts, ranks.n)
        REACHED.append({"what": ranks.what, "n_ranks": ranks.n, "rank": rank, "received": n_tuples, "limit": ranks.q.num_groups_limit,
                        **ranks.plans[rank]})
    for res in ranks.results:
        res.finalize()                    # (waits for the merge kernels: the buffers stay referenced until here)
    return [res.tables[0] for res in ranks.results]


def merged_slots(rec):
    """the least number of slots a merge gives the table it inserts into: 2 x min(numGroupsLimit, tuples received), a power of
    two of at least 1024, plus the reserved slot"""
    cap = 1024
    while cap < 2 * min(rec["limit"], max(rec["received"], 1)):
        cap *= 2
    return cap + 1


def union(tables, what):
    """the rows of all partitions, which must be pairwise disjoint"""
    rows = {}
    for rank, t in enumerate(tables):
        r = t.rows()
        assert t.num_groups == len(r), f"{what}: rank {rank}: num_groups {t.num_groups} != {len(r)} rows"
        both = set(rows) & set(r)
        assert not both, f"{what}: rank {rank} hands back groups another rank holds: {sorted(both)[:5]}"
        rows.update(r)
    return rows


def check(ranks, tables, what, limit_reached=0):
    """the union against the reference, and every rank with the statistics of the whole query"""
    rows = union(tables, what)
    assert_matches_reference(rows, ranks.ref, ranks.q, what)
    for rank, t in enumerate(tables):
        ranks.check_stats(t, f"{what}, rank {rank}")
        assert t.stats["num_groups_limit_reached"] == limit_reached, f"{what}: rank {rank}: limit flag {t.stats['num_groups_limit_reached']}"
    return rows


def _segment(name, cols):
    """cols: column -> (DataType, values, dictionary).  The segment and its reference sources."""
    built, src = [], {}
    for c, (dt, v, d) in cols.items():
        built.append(build_column(c, dt, v, dictionary=d))
        src[c] = Col(np.asarray(v).astype(np.float64 if dt in (DataType.FLOAT, DataType.DOUBLE) else np.int64), dt, d)
    return make_segment(name, built), src


def _raw_keys(name, keys, seed, extra=None):
    """a raw LONG key k, a filter column w and a metric v over the given per-doc keys"""
    r = np.random.default_rng(seed)
    n = len(keys)
    cols = {"k": (DataType.LONG, np.asarray(keys, np.int64), False), "w": (DataType.INT, r.integers(0, 2, n).astype(np.int32), True),
            "v": (DataType.INT, r.integers(-1000, 1000, n).astype(np.int32), True)}
    cols.update(extra or {})
    return _segment(name, cols)


# ---- 1: seeded fuzz ----

def _uneven(n_segs, n_ranks):
    """rank 0 holds the first segment only, the other ranks share the rest"""
    return [[0]] + [[int(i) for i in a + 1] for a in np.array_split(np.arange(n_segs - 1), n_ranks - 1)]


@pytest.mark.parametrize("seed", SEEDS)
def test_hash_fuzz_over_simulated_ranks(seed):
    segs, srcs, facts = fuzz_gen.make_tables(seed, MAX_DOCS)
    rng = np.random.default_rng(7_000 + seed)
    for qi in range(QUERIES_PER_SEED):
        sql = fuzz_gen.make_hash_query(rng, srcs[0], facts["wide_card"])
        ref = orc = None
        for ni, n in enumerate((2, 3, 4, 8)):
            if n > len(segs):
                continue
            how = ("contiguous", "interleaved", "uneven")[(qi + ni) % 3]
            parts = _uneven(len(segs), n) if how == "uneven" else None
            what = f"seed {seed} query {qi} over {n} ranks ({how}): {sql}"
            with simulate_ranks(segs, srcs, n, sql, what, interleaved=(how == "interleaved"), parts=parts) as ranks:
                assert all(p["table_mode"] == HASH for p in ranks.plans), f"{what}: {ranks.plans}"
                ranks._ref, ranks._orc = ref, orc
                check(ranks, merged_partitions(ranks), what)
                ref, orc = ranks._ref, ranks._orc           # (every shard holds all segments)


# ---- 2: functions that keep their own row count ----

def _filtered_tables(n_ranks, n=400):
    """keys 0 .. n_ranks - 1 on one rank each, 100 .. 104 on every rank; w = 1 occurs on ranks 0 and 1 only, and never for
    key 104 (its filtered functions have no input anywhere)"""
    segs, srcs = [], []
    for rank in range(n_ranks):
        r = np.random.default_rng(90 + rank)
        k = np.where(np.arange(n) % 2 == 0, rank, 100 + r.integers(0, 5, n))
        w = r.integers(0, 2, n) if rank < 2 else np.zeros(n, np.int64)
        w = np.where(k == 104, 0, w)
        s, src = _raw_keys(f"flt{rank}", k, 90 + rank, {"w": (DataType.INT, w.astype(np.int32), True)})
        segs.append(s)
        srcs.append(src)
    return segs, srcs


def test_filtered_functions_travel_with_their_own_row_counts():
    """AVG / COUNT(*) / SUM / MIN / MAX under a FILTER clause: a group the clause leaves without input on some ranks and one
    it leaves without input on all ranks.  The tuple carries the filtered row count next to the sum or min / max; without it
    the merged AVG and COUNT read 0."""
    sql = "SELECT k, AVG(v) FILTER(WHERE w = 1), COUNT(*) FILTER(WHERE w = 1), SUM(v) FILTER(WHERE w = 1), " \
          "MIN(v) FILTER(WHERE w = 1), MAX(v) FILTER(WHERE w = 1), COUNT(*), AVG(v) FROM t GROUP BY k LIMIT 100"
    for n_ranks in (2, 3, 4):
        segs, srcs = _filtered_tables(n_ranks)
        what = f"filtered functions over {n_ranks} ranks"
        with simulate_ranks(segs, srcs, n_ranks, sql, what) as ranks:
            rows = check(ranks, merged_partitions(ranks), what)
            assert rows[(104,)][1] == 0 and rows[(100,)][1] > 0, rows           # COUNT(*) FILTER


# ---- 3: enableNullHandling over a hash key ----

def test_null_handling_over_a_hash_key():
    """A raw (non-null) LONG key with nullable aggregation columns: every function keeps its input count, which reports SQL
    NULL when it is 0.  Key 0 is all-null on rank 0 only, key 1 on both ranks, key 2 on rank 1 only."""
    segs = []
    for rank, null_keys in enumerate(([0, 1], [1, 2])):
        n = 300
        k = np.arange(n) % 4
        a = (np.arange(n) % 9 + 1 + rank).astype(np.int32)
        nulls = np.isin(k, null_keys)
        segs.append(make_segment(f"hnull{rank}", [build_column("k", DataType.LONG, k.astype(np.int64), dictionary=False),
                                                  with_nulls(build_column("a", DataType.INT, np.where(nulls, INT_NULL, a).astype(np.int32)), nulls)]))
    sql = NH + "SELECT k, SUM(a), MIN(a), MAX(a), AVG(a), COUNT(a), COUNT(*) FROM t GROUP BY k LIMIT 100"
    with simulate_ranks(segs, None, 2, sql, "nulls over a hash key") as ranks:
        assert all(p["table_mode"] == HASH for p in ranks.plans), ranks.plans
        tables = merged_partitions(ranks)
        rows = union(tables, "nulls over a hash key")
        assert_rows_equal(rows, combined_rows(oracle.combine(ranks.orc), ranks.q), ranks.q, exact_float=False, what="nulls over a hash key")
        for rank, t in enumerate(tables):
            ranks.check_stats(t, f"nulls over a hash key, rank {rank}")
        assert rows[(1,)] == [None] * 4 + [0, 150]
        assert None not in rows[(0,)] and None not in rows[(2,)] and rows[(0,)][4:] == [75, 150] and rows[(2,)][4:] == [75, 150]


# ---- 4: ranks whose tables differ in size ----

def _big_rank(name, n_docs, n_keys, seed):
    r = np.random.default_rng(seed)
    keys = r.permutation(np.concatenate([np.arange(n_keys), r.integers(0, n_keys, n_docs - n_keys)])) * 7919 - 3_000_000
    return _raw_keys(name, keys, seed)


@pytest.mark.parametrize("n_ranks", [2, 4])
def test_uneven_capacities(n_ranks):
    """One rank holds a 31-doc segment (1024 slots), another 200 k docs over 100 k distinct raw keys.  The layout word does
    not cover capacity, so the merge is accepted; the small rank receives its share of 100 k groups into a table sized for
    what arrived, so no group is lost and the limit flag stays 0."""
    tables = [_raw_keys("tiny", np.arange(31) * 5, 1), _big_rank("big", 200_000, 100_000, 2)]
    tables += [_big_rank(f"mid{i}", 20_000, 15_000, 3 + i) for i in range(n_ranks - 2)]
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    sql = UNLIMITED + "SELECT k, COUNT(*), SUM(v), MAX(v), AVG(v) FILTER(WHERE w = 1) FROM t GROUP BY k LIMIT 100000000"
    with simulate_ranks(segs, srcs, n_ranks, sql, f"uneven capacities over {n_ranks} ranks") as ranks:
        rows = check(ranks, merged_partitions(ranks), f"uneven capacities over {n_ranks} ranks")
        assert len(rows) == len(ranks.ref) > 100_000


def test_merged_partition_above_2_20_slots():
    """About 600 k distinct raw keys over 2 ranks: each rank's share needs a table above 2^20 slots (the small rank's a
    grown receive table), whose hand-back counts its groups first (pb_count_groups_kernel)"""
    tables = [_raw_keys("small", np.arange(31) * 3, 5), _big_rank("large", 700_000, 600_000, 6)]
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    sql = UNLIMITED + "SELECT k, COUNT(*), SUM(v), MIN(v) FROM t GROUP BY k LIMIT 100000000"
    with simulate_ranks(segs, srcs, 2, sql, "above 2^20 slots") as ranks:
        rows = check(ranks, merged_partitions(ranks), "above 2^20 slots")
        assert len(rows) == len(ranks.ref) > 600_000
        assert min(merged_slots(r) for r in REACHED[-2:]) > 2 ** 20


# ---- 5: the reserved slot of the all-ones key ----

def test_all_ones_key_merges_into_one_group():
    """-1 is the all-ones key (PB_HASH_EMPTY) with a reserved slot (pb_sentinel_slot), in one key word and, as (-1, -1), in two"""
    segs, srcs = [], []
    for rank in range(3):
        k = np.where(np.arange(500) % 3 == 0, -1, np.arange(500) % 17 + rank)
        s, src = _raw_keys(f"ones{rank}", k, 30 + rank, {"k2": (DataType.LONG, np.where(np.arange(500) % 2 == 0, -1, 5).astype(np.int64), False)})
        segs.append(s)
        srcs.append(src)
    for sql in ("SELECT k, COUNT(*), SUM(v), MIN(v) FROM t GROUP BY k LIMIT 100",
                "SELECT k, k2, COUNT(*), SUM(v), MAX(v) FROM t GROUP BY k, k2 LIMIT 100"):
        with simulate_ranks(segs, srcs, 3, sql, f"all-ones key: {sql}") as ranks:
            rows = check(ranks, merged_partitions(ranks), f"all-ones key: {sql}")
            assert (-1,) in rows or (-1, -1) in rows


# ---- 6: empty sides ----

def test_empty_sides():
    """A rank whose filter matches nothing sends no tuples; a query with one group over four ranks leaves three ranks that
    receive nothing: they hand back 0 rows with the statistics of the whole query"""
    tables = [_raw_keys(f"e{rank}", np.arange(300) % 40 + (10_000 if rank == 1 else 0), 50 + rank) for rank in range(3)]
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    sql = "SELECT k, COUNT(*), SUM(v), MIN(v) FROM t WHERE k < 5000 GROUP BY k LIMIT 100"
    with simulate_ranks(segs, srcs, 3, sql, "a rank matches nothing") as ranks:
        assert sum(ranks.results[1].hash_partition(3)[1]) == 0
        check(ranks, merged_partitions(ranks), "a rank matches nothing")
    tables = [_raw_keys(f"one{rank}", np.full(100, 77), 60 + rank) for rank in range(4)]
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    with simulate_ranks(segs, srcs, 4, "SELECT k, COUNT(*), SUM(v), AVG(v) FROM t GROUP BY k LIMIT 100", "one group") as ranks:
        tables = merged_partitions(ranks)
        check(ranks, tables, "one group")
        assert sorted(t.num_groups for t in tables) == [0, 0, 0, 1]


# ---- 7: the order the sources arrive in ----

def test_order_independence():
    """The sources concatenated in a permuted order: counts, MIN / MAX and the key set of every rank stay bit-identical, and
    the float sums stay inside the reference's bound"""
    segs, srcs, _ = fuzz_gen.make_tables(0, 80_000)
    sql = UNLIMITED + "SELECT rki, rkj, k2, COUNT(*), SUM(mdbl), AVG(mflt), MIN(edbl), MAX(eneg), SUM(mlong), MAX(enan), " \
                      "AVG(rdbl) FILTER(WHERE fu < 900) FROM t GROUP BY rki, rkj, k2 LIMIT 100000000"
    runs = []
    for order in (None, [3, 1, 0, 2]):
        with simulate_ranks(segs, srcs, 4, sql, f"source order {order}") as ranks:
            tables = merged_partitions(ranks, order)
            check(ranks, tables, f"source order {order}")
            runs.append([_bits(t) for t in tables])
    for rank in range(4):
        _same_except_float_sums(runs[1][rank], runs[0][rank], ranks.q, f"rank {rank}: permuted source order")


# ---- 8: numGroupsLimit ----

def test_num_groups_limit_reachable_on_some_ranks():
    """numGroupsLimit = 50: rank 0 holds 300 keys and reaches it, rank 1 holds 20 and does not.  The limit-reached cells are
    summed, so every rank reports the flag.  The rule for a merged hash table: a group is handed back only if some rank
    created it, and it holds only rows that a rank aggregated (the repair pass drops every row of a refused key), so every
    group handed back is a reference key with at most the reference's row count, and no rank hands back more than the
    limit (its merge takes tickets too)."""
    tables = [_raw_keys("many", np.arange(3000) % 300, 70), _raw_keys("few", np.arange(400) % 20, 71)]
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    sql = "SET numGroupsLimit = 50; SELECT k, COUNT(*), SUM(v) FROM t GROUP BY k LIMIT 100000"
    with simulate_ranks(segs, srcs, 2, sql, "numGroupsLimit") as ranks:
        tables = merged_partitions(ranks)
        rows = union(tables, "numGroupsLimit")
        for rank, t in enumerate(tables):
            assert t.stats["num_groups_limit_reached"] == 1, f"rank {rank}"
            assert t.num_groups <= 50
            ranks.check_stats(t, f"numGroupsLimit, rank {rank}")
        assert rows
        for key, row in rows.items():
            assert key in ranks.ref and row[0] <= ranks.ref[key][0], (key, row, ranks.ref.get(key))


# ---- 9: the ORDER BY ... LIMIT trim after the merge ----

def test_trim_after_the_merge():
    """Each rank trims its own partition: the union holds every group at least as good as the reference's LIMIT-th best by
    the first ORDER BY expression (ties included), and every group handed back is exact"""
    tables = [_raw_keys(f"trim{rank}", np.random.default_rng(80 + rank).integers(0, 400, 5000), 80 + rank) for rank in range(3)]
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    opts = "SET minServerGroupTrimSize = 7; SET minSegmentGroupTrimSize = 7; SET groupTrimThreshold = 14; "
    for tail, col, sign in (("ORDER BY COUNT(*) DESC LIMIT 3", 1, 1), ("ORDER BY SUM(v) ASC LIMIT 2", 2, -1), ("ORDER BY k DESC LIMIT 4", 0, 1)):
        sql = opts + f"SELECT k, COUNT(*), SUM(v) FROM t GROUP BY k {tail}"
        limit = int(tail.split()[-1])
        with simulate_ranks(segs, srcs, 3, sql, f"trim: {tail}") as ranks:
            rows = union(merged_partitions(ranks), f"trim: {tail}")
            assert_matches_reference(rows, {k: ranks.ref[k] for k in rows}, ranks.q, f"trim: {tail}")
            exact = lambda v: v.exact if isinstance(v, SumRef) else v
            value = lambda k, row: sign * (k[0] if col == 0 else exact(row[col - 1]))
            best = sorted((value(k, r) for k, r in ranks.ref.items()), reverse=True)[limit - 1]
            want = {k for k, r in ranks.ref.items() if value(k, r) >= best}
            assert want <= set(rows), f"trim: {tail}: missing {sorted(want - set(rows))}"
            assert len(rows) < len(ranks.ref)


# ---- 10: refusals ----

def test_refusals():
    """DISTINCTCOUNT in a hash table and more than 64 ranks are refused by the partition, a dense table too; ranks that ran
    different queries (SUM vs AVG; AVG with and without a FILTER clause, whose tuples differ in width) by the merge, before it
    reads a tuple, and the results still free"""
    segs, srcs = _filtered_tables(2)
    with simulate_ranks(segs, srcs, 2, "SELECT k, DISTINCTCOUNT(v) FROM t GROUP BY k LIMIT 100", "distinct") as ranks:
        _raises(PB_ERR_UNSUPPORTED, "DISTINCTCOUNT in a hash group table is not merged across ranks", ranks.results[0].hash_partition, 2)
    with simulate_ranks(segs, srcs, 2, "SELECT k, SUM(v) FROM t GROUP BY k LIMIT 100", "65 ranks") as ranks:
        _raises(PB_ERR_UNSUPPORTED, "hash table merge over 65 ranks (max 64)", ranks.results[0].hash_partition, 65)
    with simulate_ranks(segs, srcs, 2, "SELECT w, SUM(v) FROM t GROUP BY w LIMIT 100", "dense") as ranks:
        _raises(PB_ERR_UNSUPPORTED, "a hash merge needs a combined (PB_Q_COMBINE) hash group table", ranks.results[0].hash_partition, 2)
    for a, b in (("SELECT k, SUM(v) FROM t GROUP BY k LIMIT 100", "SELECT k, AVG(v) FROM t GROUP BY k LIMIT 100"),
                 ("SELECT k, AVG(v) FROM t GROUP BY k LIMIT 100", "SELECT k, AVG(v) FILTER(WHERE w = 1) FROM t GROUP BY k LIMIT 100")):
        with simulate_ranks(segs, srcs, 2, a, f"layouts: {b}", rank_sql=[a, b]) as ranks:
            received, cells, layouts = exchange(ranks)
            assert layouts[0] != layouts[1]
            for res, (buf, n_tuples) in zip(ranks.results, received):
                _raises(PB_ERR_STATE, "table layouts differ across ranks", res.hash_merge_received, buf.data_ptr(), n_tuples, cells.data_ptr(), layouts, 2)


def test_null_vector_mismatch_is_refused():
    """enableNullHandling where one rank has a null-value vector for the aggregated column and the other none (README, open
    items): the second plans no implicit clause, so its tuples are narrower.  The merge refuses instead of misreading them."""
    segs = []
    for rank in range(2):
        k = np.arange(200) % 7
        a = (np.arange(200) % 5).astype(np.int32)
        col = build_column("a", DataType.INT, a)
        segs.append(make_segment(f"nv{rank}", [build_column("k", DataType.LONG, k.astype(np.int64), dictionary=False),
                                               with_nulls(col, k == 3) if rank == 0 else col]))
    with simulate_ranks(segs, None, 2, NH + "SELECT k, SUM(a), MIN(a) FROM t GROUP BY k LIMIT 100", "null vector mismatch") as ranks:
        received, cells, layouts = exchange(ranks)
        assert layouts[0] != layouts[1]
        for res, (buf, n_tuples) in zip(ranks.results, received):
            _raises(PB_ERR_STATE, "table layouts differ across ranks", res.hash_merge_received, buf.data_ptr(), n_tuples, cells.data_ptr(), layouts, 2)


# ---- what the module reached ----

def test_hash_merges_reached_every_shape():
    """from the merges logged by the tests above: over 2, 3, 4 and 8 ranks, with one and two key words, a rank that received
    nothing, and a merged table above 2^20 slots"""
    if os.environ.get("PB_FUZZ_SEEDS") or not any(r["what"].startswith("seed ") for r in REACHED):
        pytest.skip("needs the whole module under the default seeds")
    assert all(r["table_mode"] == HASH for r in REACHED)
    for n in (2, 3, 4, 8):
        assert any(r["n_ranks"] == n for r in REACHED), f"no hash merge over {n} ranks"
    assert {r["key_words"] for r in REACHED} == {1, 2}
    assert any(r["received"] == 0 for r in REACHED)
    assert any(merged_slots(r) > 2 ** 20 for r in REACHED)
