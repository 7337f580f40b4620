"""The cross-rank merge of group tables, held to the exact reference on ONE GPU by merging the table blocks of simulated ranks.

Several segment groups on device 0 each hold one rank's segments.  Their global dictionaries are agreed exactly as
pinot_b200/distributed.py agrees them across processes (export, merge_sorted_dictionaries, install the union), every group
runs the query with PB_Q_COMBINE | PB_Q_DEFER_FINALIZE, and the blocks (pb_result_device_buffer(which = 8)) are copied
rank-major into one buffer: what an all-gather would deliver.  pb_result_merge_gathered + pb_result_finalize then run the real
pb_merge_blocks_kernel, the real local-to-global remaps and the real hand-back over a merged table, and the result is judged by
tests/reference.py over all segments of all ranks.

Not covered here: NCCL itself (comm_merge's collectives) and the pointer plumbing of the NVLink peer merge.  The
hash-partitioned all-to-all of hash tables is held to the reference the same way in tests/test_gpu_hash_merge.py.

PB_FUZZ_SEEDS="1,3" narrows the fuzz seeds."""
import contextlib
import itertools
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from pinot_b200 import native
from pinot_b200.distributed import dictionary_columns, merge_sorted_dictionaries
from pinot_b200.query import AggOp, parse_sql
from pinot_b200.segment_writer import DataType, build_column, make_segment, with_nulls
from tests import fuzz_gen
from tests.parity import assert_rows_equal, combined_rows
from tests.reference import Col, assert_matches_reference, concat, limit_reference, reference
from tests.test_cpu_null_handling import INT_NULL, NH
from tests.test_gpu_fuzz import _carry_table, _group
from tests.test_gpu_null_handling import FUZZ_QUERIES as NULL_QUERIES, fuzz_segments as null_segments
from tests.test_gpu_result_shaping import check_table

pytestmark = pytest.mark.gpu

# seed 1: 24 segments (4 ranks hold several each); seed 3: 5 segments, a rank that holds one 31-doc segment only; seed 2: 4097
# values in kwb (kwa, kwb is a hash table)
SEEDS = [int(s) for s in os.environ["PB_FUZZ_SEEDS"].split(",")] if os.environ.get("PB_FUZZ_SEEDS") else [1, 2, 3]
QUERIES_PER_SEED = 5
MAX_DOCS = 200_000
PB_ERR_INVALID, PB_ERR_UNSUPPORTED, PB_ERR_STATE = -1, -2, -5
KEYLESS, DENSE, HASH = 0, 1, 2
DEFERRED = native.PB_Q_COMBINE | native.PB_Q_DEFER_FINALIZE
REACHED = []                    # one record per simulated rank: what, n_ranks, rank, slots, merged + its plan_info


@pytest.fixture(scope="module", autouse=True)
def _device():
    native.init()
    yield
    torch.cuda.empty_cache()


# ---- the harness ----

class _DevicePointer:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def device_view(ptr: int, nbytes: int) -> torch.Tensor:
    """zero-copy uint8 view of device memory the library owns"""
    return torch.as_tensor(_DevicePointer(ptr, nbytes), device="cuda")


def shard(n_segs, n_ranks, interleaved=False):
    """contiguous shards, or the round-robin of distributed.shard_segments"""
    if interleaved:
        return [list(range(r, n_segs, n_ranks)) for r in range(n_ranks)]
    return [[int(i) for i in a] for a in np.array_split(np.arange(n_segs), n_ranks)]


class Ranks:
    """n simulated ranks on device 0: parts[r] = the indexes (into segs / srcs) of rank r's segments"""

    def __init__(self, segs, srcs, parts, sql, what, rank_flags=None, rank_sql=None):
        assert all(parts), f"{what}: a rank without segments: {parts}"
        self.segs, self.srcs, self.parts, self.what = segs, srcs, parts, what
        self.n = len(parts)
        self.queries = [parse_sql(s) for s in (rank_sql or [sql] * self.n)]
        self.q = self.queries[0]
        self.flags = rank_flags or [0] * self.n
        self.staged, self.groups, self.results, self.plans = [], [], [], []
        self.slots = 1
        self._ref = self._orc = None

    def used(self, xs):
        return [xs[i] for p in self.parts for i in p]

    @property
    def ref(self):
        if self._ref is None:
            self._ref = reference(concat(self.used(self.srcs)), self.q)
        return self._ref

    @property
    def orc(self):
        if self._orc is None:
            self._orc = [oracle.execute(s, self.q) for s in self.used(self.segs)]
        return self._orc

    def stage(self):
        for p in self.parts:
            st, g = _group([self.segs[i] for i in p])
            self.staged.append(st)
            self.groups.append(g)

    def agree(self):
        """the union over all ranks of every dictionary the tables are laid out by, installed in every group"""
        seg0 = self.segs[self.parts[0][0]]
        cols = []
        for q in self.queries:
            cols += [c for c in dictionary_columns(q, seg0) if c not in cols]
        for c in cols:
            union = merge_sorted_dictionaries([g.export_dictionary(c) for g in self.groups], int(seg0.columns[c].data_type))
            for g in self.groups:
                g.set_global_dictionary(c, union)
            if c in self.q.group_by:
                self.slots *= len(union)

    def execute(self):
        for r, (g, q, f) in enumerate(zip(self.groups, self.queries, self.flags)):
            res = native.execute(g, q, DEFERRED | f)
            self.results.append(res)
            res.wait()
            self.plans.append(res.plan_info)
            REACHED.append({"what": self.what, "n_ranks": self.n, "rank": r, "slots": self.slots, "merged": False, **res.plan_info})

    def blocks(self, results=None):
        """(device pointer, bytes) of every rank's table block; the sizes must agree before anything is copied"""
        blocks = [res.device_buffer(8) for res in (results or self.results)]
        assert len({n for _, n in blocks}) == 1, f"{self.what}: block sizes differ across ranks: {[n for _, n in blocks]}"
        return blocks

    def gather(self, order=None, results=None):
        """what an all-gather over the ranks `order` delivers: their blocks, rank-major, in one device buffer"""
        blocks = self.blocks(results)
        order = list(range(len(blocks))) if order is None else order
        size = blocks[0][1]
        buf = torch.empty(len(order) * size, dtype=torch.uint8, device="cuda")
        for i, r in enumerate(order):
            buf[i * size:(i + 1) * size].copy_(device_view(blocks[r][0], size))
        torch.cuda.synchronize()
        return buf

    def merge(self, rank, buf, n_rows):
        self.results[rank].merge_gathered(buf.data_ptr(), n_rows)
        for rec in REACHED[-self.n:]:
            rec["merged"] = True

    def merged_table(self, into=0, order=None):
        """gather, merge into one rank's result, finalize: its table"""
        buf = self.gather(order)
        self.merge(into, buf, self.n)
        self.results[into].finalize()           # (waits for the merge kernel: buf stays referenced until here)
        return self.results[into].tables[0]

    def check_stats(self, t, what):
        for key in ("num_docs_scanned", "num_total_docs", "num_entries_scanned_post_filter"):
            exp = sum(o.stats[key] for o in self.orc)
            assert t.stats[key] == exp, f"{what}: {key}: {t.stats[key]} != {exp} over all ranks"
        assert t.stats["num_total_docs"] == sum(s.num_docs for s in self.used(self.segs)), what
        assert t.stats["num_segments"] == sum(len(p) for p in self.parts), f"{what}: num_segments {t.stats['num_segments']}"

    def check(self, t, what):
        assert_matches_reference(t.rows(), self.ref, self.q, what)
        self.check_stats(t, what)

    def release(self):
        for res in self.results:
            res.free()
        for g in self.groups:
            g.release()
        for st in self.staged:
            for s in st:
                s.release()


@contextlib.contextmanager
def simulate_ranks(segs, srcs, n_ranks, sql, what="", interleaved=False, parts=None, rank_flags=None, rank_sql=None):
    """The ranks with their dictionaries agreed and their deferred results computed; everything is released on exit."""
    ranks = Ranks(segs, srcs, parts or shard(len(segs), n_ranks, interleaved), sql, what, rank_flags, rank_sql)
    try:
        ranks.stage()
        ranks.agree()
        ranks.execute()
        yield ranks
    finally:
        ranks.release()


def _raises(code, message, fn, *args):
    with pytest.raises(native.PinotB200Error) as e:
        fn(*args)
    assert e.value.code == code and message in str(e.value), f"expected error {code} '{message}', got: {e.value}"


def _raw_distinct(q, seg):
    return any(a.op == AggOp.DISTINCTCOUNT and not seg.columns[a.column].has_dictionary for a in q.aggregations)


def merge_or_refusal(ranks, into=0):
    """The merged table of a keyless / dense query, or None after checking the documented refusals: a hash table exposes no
    block, and a DISTINCTCOUNT over a raw column is not merged."""
    modes = {p["table_mode"] for p in ranks.plans}
    assert len(modes) == 1, f"{ranks.what}: ranks disagree on the table mode: {ranks.plans}"
    if modes == {HASH}:
        for res in ranks.results:
            _raises(PB_ERR_UNSUPPORTED, "hash tables cannot be all-reduced in place", res.device_buffer, 8)
        return None
    if _raw_distinct(ranks.q, ranks.segs[0]):
        buf = ranks.gather()
        _raises(PB_ERR_UNSUPPORTED, "DISTINCTCOUNT on a raw column is not merged across GPUs", ranks.results[into].merge_gathered,
                buf.data_ptr(), ranks.n)
        return None
    return ranks.merged_table(into)


def _bits(t):
    """key -> per aggregation (double as int64 bits, long): the long of COUNT, DISTINCTCOUNT and AVG, the double of the rest
    and of AVG (what the hand-back defines)"""
    keys = t.keys() if t.query.group_by else [()]
    ops = [a.op for a in t.query.aggregations]
    return {k: [(0 if op in (AggOp.COUNT, AggOp.DISTINCTCOUNT) else int(np.asarray(t.doubles[a][g]).view(np.int64)),
                 int(t.longs[a][g]) if op in (AggOp.COUNT, AggOp.DISTINCTCOUNT, AggOp.AVG) else 0) for a, op in enumerate(ops)]
            for g, k in enumerate(keys)}


def _same_except_float_sums(a, b, q, what):
    assert set(a) == set(b), f"{what}: group sets differ"
    for k in a:
        for i, agg in enumerate(q.aggregations):
            if agg.op in (AggOp.SUM, AggOp.AVG):
                assert a[k][i][1] == b[k][i][1], f"{what}: {k} {agg}: counts {a[k][i][1]} != {b[k][i][1]}"
            else:
                assert a[k][i] == b[k][i], f"{what}: {k} {agg}: {a[k][i]} != {b[k][i]}"


# ---- 1: seeded fuzz ----

@pytest.mark.parametrize("seed", SEEDS)
def test_fuzz_over_simulated_ranks(seed):
    segs, srcs, _ = fuzz_gen.make_tables(seed, MAX_DOCS)
    rng = np.random.default_rng(5_000 + seed)
    for qi in range(QUERIES_PER_SEED):
        sql = fuzz_gen.make_query(rng, srcs[0])
        ref = orc = None
        for n in (2, 3, 4):
            # (2^24 slots: the gathered buffer is ranks x slots x 8 x (1 + aggregations) bytes)
            if n > len(segs) or (n > 2 and "kwa" in sql.split("GROUP BY")[-1]):
                continue
            what = f"seed {seed} query {qi} over {n} ranks: {sql}"
            with simulate_ranks(segs, srcs, n, sql, what, interleaved=(n == 3 and qi % 2 == 1)) as ranks:
                ranks._ref, ranks._orc = ref, orc
                t = merge_or_refusal(ranks, into=qi % n)
                if t is not None:
                    ranks.check(t, what)
                ref, orc = ranks._ref, ranks._orc           # the same segments under every rank count


# ---- 2: ranks on different kernel paths ----

def _with_f(seg, src, f):
    """the segment with its filter column f replaced"""
    cols = [build_column("f", DataType.INT, f.astype(np.int32))] + [c for name, c in seg.columns.items() if name != "f"]
    return make_segment(seg.name + "_f", cols), {**src, "f": Col(f.astype(np.int64), DataType.INT)}


def test_ranks_on_different_kernel_paths_produce_one_layout():
    """One query, four ranks: the fused filter kernel (a selective leaf), pb_agg_rows_kernel with a CTA table and exact-integer
    sums (2 M docs, a third of them kept), the general filter kernel, and a rank whose filter matches nothing (it ships a
    table of initial cells).  The layout fingerprints agree and the merged INT sums are the exact integer sums (the
    reference demands it: docs x 2^31 < 2^53)."""
    r = np.random.default_rng(2)
    tables = [_with_f(*_carry_table(60_000, seed=6), r.integers(0, 400, 60_000)),      # f = 0 keeps 1 / 400
              _carry_table(2_000_000),
              _carry_table(50_000, seed=7),
              _with_f(*_carry_table(10_000, seed=8), np.ones(10_000, np.int64))]      # no doc has f = 0
    segs, srcs = [t[0] for t in tables], [t[1] for t in tables]
    sql = "SELECT k, COUNT(*), SUM(vi), AVG(vi), MIN(vi), MAX(vi), MAX(neg), MIN(pos), MIN(nan), MAX(nan) FROM t " \
          "WHERE f = 0 AND pos < 100 GROUP BY k LIMIT 100"
    flags = [0, 0, native.PB_Q_GENERIC_KERNEL, 0]
    with simulate_ranks(segs, srcs, 4, sql, "kernel paths", rank_flags=flags) as ranks:
        fused, rows, general, empty = ranks.plans
        assert fused["fused_agg"] == 1, ranks.plans
        if os.environ.get("PB_AGG_SMEM", "1") != "0":
            assert rows["agg_kernel"] == 3 and rows["fused_agg"] == 0 and rows["st_replicas"] > 0 and rows["exact_int_mask"] == 0b110, ranks.plans
        assert general["filter_kernel"] in (1, 2), ranks.plans
        assert reference(srcs[3], ranks.q) == {}
        t = ranks.merged_table()
        ranks.check(t, "kernel paths")
        assert len(t.rows()) == 4


# ---- 3: region edges of the block ----

def _edge_table(n_ranks=3, n=600):
    """keys below n_ranks: each on one rank only; keys n_ranks .. n_ranks + 2: on every rank.  e: group 0 every edge double, group 1 the two zeros, group 2
    the two infinities, the first shared group NaN only.  w = 1 (the FILTER clauses) occurs on ranks 0 and 1 only."""
    segs, srcs = [], []
    E = fuzz_gen.EDGE_DOUBLES
    for rank in range(n_ranks):
        r = np.random.default_rng(40 + rank)
        k = np.where(np.arange(n) % 2 == 0, rank, n_ranks + r.integers(0, 3, n))
        e_ids = r.integers(0, len(E), n)
        e_ids = np.where(k == 1, 4 + r.integers(0, 2, n), e_ids)           # -0.0, 0.0
        e_ids = np.where(k == 2, np.where(r.integers(0, 2, n) == 0, 0, 10), e_ids)       # -inf, inf
        e_ids = np.where(k == n_ranks, 11, e_ids)                                                # NaN
        w = r.integers(0, 2, n) if rank < 2 else np.zeros(n, np.int64)
        v = r.integers(-1000, 1000, n)
        cols = [build_column("k", DataType.INT, k.astype(np.int32)), build_column("w", DataType.INT, w.astype(np.int32)),
                build_column("v", DataType.INT, v.astype(np.int32))]
        src = {"k": Col(k.astype(np.int64), DataType.INT), "w": Col(w.astype(np.int64), DataType.INT), "v": Col(v, DataType.INT)}
        for name, d, ids in (("e", E, e_ids), ("neg", fuzz_gen.NEG_DOUBLES, r.integers(0, len(fuzz_gen.NEG_DOUBLES), n)),
                             ("nan", np.array([np.nan]), np.zeros(n, np.int64))):
            cols.append(fuzz_gen._dict_col(name, DataType.DOUBLE, d, ids))
            src[name] = fuzz_gen._src(DataType.DOUBLE, d, ids)
        segs.append(make_segment(f"edge{rank}", cols))
        srcs.append(src)
    return segs, srcs


def test_initial_cells_are_neutral_and_empty_regions_merge():
    """MIN / MAX where only one rank has input for a group (the others ship the initial cell, neutral under the i64 MIN for the
    MIN table and for the bit-complemented MAX table), queries whose f64 and / or min-max regions are empty, a keyless block,
    and FILTER clauses that leave a rank no input"""
    for n_ranks, sql in itertools.product((2, 3, 4), ("SELECT k, MIN(e), MAX(e), MIN(neg), MAX(neg), MIN(nan), MAX(nan) FROM t GROUP BY k LIMIT 100",        # no f64 region
                "SELECT k, COUNT(*) FROM t GROUP BY k LIMIT 100",                                                    # counts only
                "SELECT k, MIN(e) FROM t WHERE v < 0 GROUP BY k LIMIT 100",
                "SELECT MIN(e), MAX(e), MAX(neg), MIN(nan), COUNT(*), SUM(v) FROM t",                                 # keyless
                "SELECT COUNT(*) FROM t WHERE v > 5000",                                                              # keyless, no match
                "SELECT k, SUM(v) FILTER(WHERE w = 1), MIN(e) FILTER(WHERE w = 1), MAX(neg) FILTER(WHERE w = 1), "
                "COUNT(*) FILTER(WHERE w = 1), AVG(v), COUNT(*) FROM t GROUP BY k LIMIT 100")):
        segs, srcs = _edge_table(n_ranks)
        for order in (None, list(range(n_ranks))[::-1]):
            with simulate_ranks(segs, srcs, n_ranks, sql, f"edges: {sql}") as ranks:
                ranks.check(ranks.merged_table(order=order), f"edges over {n_ranks} ranks, order {order}: {sql}")


@pytest.mark.parametrize("width", [31, 32, 33, 65])
def test_distinct_bitsets_or_across_ranks_at_word_edges(width):
    """DISTINCTCOUNT over a dictionary column whose per-rank dictionaries are disjoint (ranks 0 and 1), overlapping (rank 2
    with both) and a strict subset (rank 3 of rank 0), their union `width` values wide: the bitset words of the OR region.
    Three groups x an odd number of 32-bit words puts a half-filled 64-bit word at the end of a bitset."""
    universe = np.arange(width, dtype=np.int64) * 7 - 20
    h = width // 2
    dicts = [universe[:h], universe[h:], universe[h - 3:h + 3], universe[:2]]
    segs, srcs = [], []
    for rank, d in enumerate(dicts):
        r = np.random.default_rng(60 + rank)
        n = 40 * len(d)
        ids = r.permutation(np.arange(n) % len(d))             # every entry occurs
        k = r.integers(0, 3, n)
        s = r.integers(0, 5, n) + rank
        segs.append(make_segment(f"dc{rank}", [build_column("k", DataType.INT, k.astype(np.int32)), fuzz_gen._dict_col("d", DataType.LONG, d, ids),
                                               build_column("s", DataType.INT, s.astype(np.int32))]))
        srcs.append({"k": Col(k.astype(np.int64), DataType.INT), "d": fuzz_gen._src(DataType.LONG, d, ids), "s": Col(s.astype(np.int64), DataType.INT)})
    for sql in ("SELECT k, DISTINCTCOUNT(d), COUNT(*), DISTINCTCOUNT(s) FROM t GROUP BY k LIMIT 100",
                "SELECT DISTINCTCOUNT(d), DISTINCTCOUNT(s) FROM t WHERE s > 1"):
        with simulate_ranks(segs, srcs, 4, sql, f"bitsets {width}: {sql}") as ranks:
            t = ranks.merged_table(into=3)
            ranks.check(t, f"bitsets {width}: {sql}")
            if not ranks.q.group_by and "WHERE" not in sql:
                assert t.rows()[()][0] == width


# ---- 4: every rank computes the same bits ----

def test_every_rank_computes_the_same_bits():
    """The same gathered buffer merged into each rank's result gives bit-identical tables (sums are added in row order).
    With the rank order of the buffer permuted, counts, MIN / MAX and DISTINCTCOUNT stay identical and the float sums stay
    inside the reference's bound."""
    segs, srcs, _ = fuzz_gen.make_tables(0, 80_000)
    sql = "SELECT k3, kstr, COUNT(*), SUM(mdbl), AVG(mflt), MIN(edbl), MAX(eneg), DISTINCTCOUNT(mint), SUM(mlong), MAX(enan) " \
          "FROM t WHERE fu < 1500 GROUP BY k3, kstr LIMIT 100000"
    with simulate_ranks(segs, srcs, 4, sql, "same bits") as ranks:
        buf = ranks.gather()
        tables = []
        for rank in range(4):
            ranks.merge(rank, buf, 4)
            ranks.results[rank].finalize()
            tables.append(ranks.results[rank].tables[0])
        ranks.check(tables[0], "same bits")
        first = _bits(tables[0])
        for rank in range(1, 4):
            assert _bits(tables[rank]) == first, f"rank {rank}'s merged table differs from rank 0's"
            assert tables[rank].stats == tables[0].stats
    with simulate_ranks(segs, srcs, 4, sql, "same bits, permuted") as ranks:
        t = ranks.merged_table(into=2, order=[3, 1, 0, 2])
        ranks.check(t, "permuted rank order")
        _same_except_float_sums(_bits(t), first, ranks.q, "permuted rank order")


# ---- 5: the merged group count ----

def _keyed_tables(card, n_keys, how, n_ranks=3, seed=0):
    """three ranks of docs over keys (ka, kb), each a full dictionary of `card` values; `how`: every rank holds the same keys,
    disjoint keys, or half and half"""
    r = np.random.default_rng(seed)
    pairs = r.choice(card * card, n_keys, replace=False)
    dv = np.arange(card, dtype=np.int64) * 3
    segs, srcs = [], []
    for rank in range(n_ranks):
        own = pairs[rank::n_ranks]
        mine = pairs if how == "same" else own if how == "disjoint" else np.concatenate([pairs[:n_keys // 2], own])
        p = r.permutation(np.concatenate([mine, mine[:len(mine) // 3]]))         # a third of the keys twice
        v = r.integers(-100, 100, len(p))
        cols, src = [build_column("v", DataType.INT, v.astype(np.int32))], {"v": Col(v, DataType.INT)}
        for name, ids in (("ka", p // card), ("kb", p % card)):
            cols.append(fuzz_gen._dict_col(name, DataType.INT, dv, ids))
            src[name] = fuzz_gen._src(DataType.INT, dv, ids)
        segs.append(make_segment(f"keys{rank}", cols))
        srcs.append(src)
    return segs, srcs


@pytest.mark.parametrize("card", [300, 1100], ids=["below 2^20 slots", "above 2^20 slots"])
def test_groups_on_several_ranks_are_counted_once(card):
    """num_groups and the rows handed back equal the reference's group count when the ranks hold the same keys, disjoint
    keys and a mix.  The merge sums counter cell [0] over the ranks, so nothing after a merge may take it for a group count;
    a table above 2^20 slots sizes its host arrays by a count of its own."""
    sql = "SET numGroupsLimit = 100000000; SELECT ka, kb, COUNT(*), SUM(v), MAX(v) FROM t GROUP BY ka, kb LIMIT 100000000"
    for how in ("same", "disjoint", "mix"):
        segs, srcs = _keyed_tables(card, 3_000, how)
        with simulate_ranks(segs, srcs, 3, sql, f"group count {card} {how}") as ranks:
            assert ranks.slots == card * card and all(p["table_mode"] == DENSE for p in ranks.plans), (ranks.slots, ranks.plans)
            t = ranks.merged_table(into=1)
            assert t.num_groups == len(ranks.ref) and len(t.rows()) == len(ranks.ref), \
                f"{card} {how}: {t.num_groups} groups, {len(t.rows())} rows, reference {len(ranks.ref)}"
            ranks.check(t, f"group count {card} {how}")
            assert t.stats["num_groups_limit_reached"] == 0


# ---- 6: result shaping after a merge ----

def _check_shaped(ranks, t, what):
    lref = limit_reference(concat(ranks.used(ranks.srcs)), ranks.q, "merged", ranks.slots)
    check_table(t, lref, ranks.q, True, what)
    ranks.check_stats(t, what)


@pytest.mark.parametrize("seed", [s for s in SEEDS if s != 2])
def test_shaped_fuzz_over_simulated_ranks(seed):
    """numGroupsLimit and the ORDER BY ... LIMIT trim over a merged dense table: the trim ranks the merged aggregates"""
    segs, srcs, _ = fuzz_gen.make_tables(seed, MAX_DOCS)
    rng = np.random.default_rng(6_000 + seed)
    for qi in range(QUERIES_PER_SEED):
        sql = fuzz_gen.make_shaped_query(rng, srcs[0])
        for n in (2, 4) if qi % 2 else (3,):
            if n > len(segs) or (n > 2 and "kwa" in sql.split("GROUP BY")[-1]):
                continue
            what = f"shaped seed {seed} query {qi} over {n} ranks: {sql}"
            with simulate_ranks(segs, srcs, n, sql, what) as ranks:
                t = merge_or_refusal(ranks, into=n - 1)
                if t is not None:
                    _check_shaped(ranks, t, what)


def test_trim_orders_by_the_merged_average():
    """ORDER BY AVG(v) where rank 0 holds a few large values per group and rank 1 many small ones, in opposite orders: the
    best groups by either rank's partial average are not the best by the merged one.  Also under a numGroupsLimit that each
    (single-segment) rank reaches on its own."""
    groups = 40
    k0 = np.repeat(np.arange(groups), 2)
    v0 = 1000 + 50 * k0                                   # rank 0 alone: group 39 is best
    k1 = np.repeat(np.arange(groups), 2 + 2 * (np.arange(groups) % 7))
    v1 = (groups - k1) * 3                                # rank 1 alone: group 0 is best
    segs, srcs = [], []
    for name, k, v in (("avg0", k0, v0), ("avg1", k1, v1)):
        p = np.random.default_rng(len(k)).permutation(len(k))
        segs.append(make_segment(name, [build_column("k", DataType.INT, k[p].astype(np.int32)), build_column("v", DataType.INT, v[p].astype(np.int32))]))
        srcs.append({"k": Col(k[p].astype(np.int64), DataType.INT), "v": Col(v[p].astype(np.int64), DataType.INT)})
    opts = "SET minServerGroupTrimSize = 7; SET minSegmentGroupTrimSize = 7; SET groupTrimThreshold = 14; "
    for pre in ("", "SET numGroupsLimit = 12; "):
        for tail in ("ORDER BY AVG(v) DESC LIMIT 1", "ORDER BY AVG(v) ASC LIMIT 1", "ORDER BY SUM(v) DESC LIMIT 1", "ORDER BY k DESC LIMIT 1"):
            sql = pre + opts + f"SELECT k, AVG(v), SUM(v), COUNT(*) FROM t GROUP BY k {tail}"
            with simulate_ranks(segs, srcs, 2, sql, f"merged average: {sql}") as ranks:
                _check_shaped(ranks, ranks.merged_table(into=1), f"merged average: {sql}")


# ---- 7: two-level merge ----

def test_two_level_merge_equals_the_flat_one():
    """4 ranks as 2 x 2: the pairs are merged, then the two merged blocks.  merged_ranks multiplies to 4, which the
    fingerprint check demands, and every non-float column equals the flat 4-rank merge bit for bit."""
    segs, srcs, _ = fuzz_gen.make_tables(4, 80_000)
    sql = "SELECT k2, k3, COUNT(*), SUM(mint), AVG(mdbl), MIN(edbl), MAX(mlong), DISTINCTCOUNT(kstr), COUNT(*) FILTER(WHERE fu < 900) " \
          "FROM t WHERE finv < 150 GROUP BY k2, k3 LIMIT 100"
    with simulate_ranks(segs, srcs, 4, sql, "flat merge") as ranks:
        t = ranks.merged_table()
        ranks.check(t, "flat 4-rank merge")
        flat = _bits(t)
    with simulate_ranks(segs, srcs, 4, sql, "two-level merge") as ranks:
        for pair in ([0, 1], [2, 3]):
            buf = ranks.gather(order=pair)
            ranks.merge(pair[0], buf, 2)
            ranks.results[pair[0]].wait()
        heads = [ranks.results[0], ranks.results[2]]
        buf = ranks.gather(results=heads)
        ranks.merge(0, buf, 2)
        ranks.results[0].finalize()
        t = ranks.results[0].tables[0]
        ranks.check(t, "two-level merge")
        _same_except_float_sums(_bits(t), flat, ranks.q, "two-level vs flat")


# ---- 8: the layout fingerprint ----

@pytest.mark.parametrize("a,b", [("SELECT k2, k3, COUNT(*), SUM(mint) FROM t GROUP BY k2, k3 LIMIT 100", "SELECT k3, k2, COUNT(*), SUM(mint) FROM t GROUP BY k3, k2 LIMIT 100"),
                                 ("SELECT k3, SUM(mint), MAX(mdbl) FROM t GROUP BY k3 LIMIT 100", "SELECT k3, AVG(mint), MAX(mdbl) FROM t GROUP BY k3 LIMIT 100"),
                                 ("SELECT k3, MIN(mint) FROM t GROUP BY k3 LIMIT 100", "SELECT k3, MAX(mint) FROM t GROUP BY k3 LIMIT 100")],
                         ids=["key order", "SUM vs AVG", "MIN vs MAX"])
def test_fingerprint_rejects_blocks_of_another_layout(a, b):
    """Two ranks whose blocks have the same size and a different layout: finalize fails with PB_ERR_STATE and the results can
    still be freed.  The same query on both ranks is accepted.  (Blocks of different sizes are never merged: Ranks.blocks.)"""
    segs, srcs, _ = fuzz_gen.make_tables(6, 20_000)
    with simulate_ranks(segs, srcs, 2, a, "fingerprint", rank_sql=[a, b]) as ranks:
        buf = ranks.gather()
        ranks.merge(0, buf, 2)
        _raises(PB_ERR_STATE, "table layouts differ across ranks", ranks.results[0].finalize)
    with simulate_ranks(segs, srcs, 2, a, "fingerprint, same query") as ranks:
        ranks.check(ranks.merged_table(), "fingerprint, same query")


# ---- 9: a global dictionary installed after the group has run ----

def test_global_dictionary_installed_after_the_group_has_run():
    """Two segments with the same key dictionary: the remaps are the identity and the kernels get none.  After three runs (a
    cached plan and its CUDA graph), a larger union dictionary is installed: the remaps stop being the identity, the cached
    plan must be retired, and the same SQL still matches the reference per segment, combined, and deferred."""
    dv = np.arange(20, dtype=np.int64) * 10
    segs, srcs = [], []
    for si, n in enumerate((30_000, 7_000)):
        r = np.random.default_rng(70 + si)
        ids, f, v = r.integers(0, 20, n), r.integers(0, 2, n), r.integers(-500, 500, n)
        segs.append(make_segment(f"late{si}", [fuzz_gen._dict_col("k", DataType.INT, dv, ids), build_column("f", DataType.INT, f.astype(np.int32)),
                                               build_column("v", DataType.INT, v.astype(np.int32))]))
        srcs.append({"k": fuzz_gen._src(DataType.INT, dv, ids), "f": Col(f, DataType.INT), "v": Col(v, DataType.INT)})
    sql = "SELECT k, COUNT(*), SUM(v), MIN(v) FROM t WHERE f = 0 GROUP BY k LIMIT 100"
    q = parse_sql(sql)
    ref_all, ref_seg = reference(concat(srcs), q), [reference(s, q) for s in srcs]
    staged, g = _group(segs)
    results = []

    def run(flags, what):
        res = native.execute(g, q, flags)
        results.append(res)
        if flags & native.PB_Q_DEFER_FINALIZE:
            res.wait()
            res.finalize()
        refs = [ref_all] if flags & native.PB_Q_COMBINE else ref_seg
        assert len(res.tables) == len(refs)
        for t, ref in zip(res.tables, refs):
            assert_matches_reference(t.rows(), ref, q, f"{what} flags={flags}")
        res.free()
    try:
        for rep in range(3):
            run(native.PB_Q_COMBINE, f"before the install, run {rep}")
        for si in range(2):
            assert (g.remap("k", si) == np.arange(20)).all()
        union = merge_sorted_dictionaries([g.export_dictionary("k"), (np.arange(15, dtype=np.int32) * 20 - 95).view(np.uint8).reshape(-1, 4)], 0)
        assert len(union) == 35
        g.set_global_dictionary("k", union)
        for si in range(2):
            rm = g.remap("k", si)
            assert len(rm) == 20 and not (rm == np.arange(20)).all() and (union.view(np.int32).reshape(-1)[rm] == dv).all()
        for rep in range(2):
            run(native.PB_Q_COMBINE, f"after the install, run {rep}")
            run(0, f"after the install, per segment, run {rep}")
            run(DEFERRED, f"after the install, deferred, run {rep}")
    finally:
        for res in results:
            res.free()
        g.release()
        for s in staged:
            s.release()


# ---- 10: enableNullHandling across ranks ----

def _check_nulls(ranks, t, what, check_stats=True):
    exp = combined_rows(oracle.combine(ranks.orc), ranks.q)
    assert_rows_equal(t.rows(), exp, ranks.q, exact_float=False, what=what)
    if check_stats:
        ranks.check_stats(t, what)


def test_null_handling_across_ranks():
    """The per-aggregation input counts travel in the block: two queries of the null-handling fuzz over two ranks against the
    oracle's cross-segment merge, and a group whose inputs are all null on one rank and not on the other.  (The segment
    without null-value vectors shares a rank with one that has them: a rank none of whose segments has a null-value vector
    for a column lays out a smaller block, which no merge accepts -- README, open items.)"""
    segs = null_segments()
    for sql in (NULL_QUERIES[0], NULL_QUERIES[1]):
        with simulate_ranks(segs, None, 2, NH + sql, f"nulls: {sql}", parts=[[0, 1], [2]]) as ranks:
            _check_nulls(ranks, ranks.merged_table(into=1), f"nulls: {sql}")
    segs = []
    for rank, null_keys in enumerate(([0, 1], [1, 2])):           # key 0: null on rank 0 only; key 1: on both; key 2: on rank 1 only
        n = 300
        k = np.arange(n) % 4
        a = (np.arange(n) % 9 + 1 + rank).astype(np.int32)
        nulls = np.isin(k, null_keys)
        segs.append(make_segment(f"allnull{rank}", [build_column("k", DataType.INT, k.astype(np.int32)),
                                                    with_nulls(build_column("a", DataType.INT, np.where(nulls, INT_NULL, a).astype(np.int32)), nulls)]))
    sql = NH + "SELECT k, SUM(a), MIN(a), MAX(a), AVG(a), COUNT(a), COUNT(*) FROM t GROUP BY k LIMIT 100"
    with simulate_ranks(segs, None, 2, sql, "all-null group") as ranks:
        t = ranks.merged_table()
        _check_nulls(ranks, t, "all-null group")
        rows = t.rows()
        assert rows[(1,)] == [None] * 4 + [0, 150]
        assert None not in rows[(0,)] and None not in rows[(2,)] and rows[(0,)][4:] == [75, 150] and rows[(2,)][4:] == [75, 150]


# ---- 11: the device buffers a caller may ask for ----

def test_only_the_whole_block_is_exposed():
    """pb_result_device_buffer hands out the whole table block (which = 8) and nothing else: the per-region buffers for a
    caller's all-reduce were removed (an all-reduce sums the fingerprint cell without telling the result how many ranks went in,
    so finalize always refused the merged table)"""
    segs, srcs, _ = fuzz_gen.make_tables(6, 20_000)
    with simulate_ranks(segs, srcs, 2, "SELECT k3, COUNT(*), SUM(mint), MIN(mdbl), DISTINCTCOUNT(fu) FROM t GROUP BY k3 LIMIT 100", "buffers") as ranks:
        res = ranks.results[0]
        for which in (0, 1, 2, 3, 4, 5, 6, 7, 9, -1):
            _raises(PB_ERR_INVALID, "no such device buffer", res.device_buffer, which, 1)
        ptr, size = res.device_buffer(8)
        assert ptr and size > 0 and size % 8 == 0
        assert res.stream() != 0
        ranks.check(ranks.merged_table(), "buffers")


# ---- what the module reached ----

def test_merges_reached_every_shape():
    """from the plans logged by the tests above: keyless and dense tables were merged over 2, 3 and 4 ranks, a dense table
    above 2^20 slots too, and a hash table was refused"""
    if os.environ.get("PB_FUZZ_SEEDS") or not any(r["what"].startswith("seed ") for r in REACHED):
        pytest.skip("needs the whole module under the default seeds")
    merged = [r for r in REACHED if r["merged"]]
    for mode in (KEYLESS, DENSE):
        for n in (2, 3, 4):
            assert any(r["table_mode"] == mode and r["n_ranks"] == n for r in merged), f"no merge of table mode {mode} over {n} ranks"
    assert any(r["table_mode"] == DENSE and r["slots"] > 2 ** 20 for r in merged)
    assert any(r["table_mode"] == HASH for r in REACHED if not r["merged"])
    assert any(r["fused_agg"] for r in merged)
    assert any(r["agg_kernel"] == 3 and r["st_replicas"] > 0 and not r["fused_agg"] for r in merged)
    assert any(r["filter_kernel"] in (1, 2) for r in merged)
