"""The device's decoders of a segment's storage formats, held to the exact reference (tests/reference.py) and the oracle
at the edges of each format:

A. RoaringBitmap blobs of inverted indexes and null-value vectors (pb_expand_kernel): array, bitmap and run containers,
   cookies 12346 and 12347, the offset header (4 or more containers) and the walk over the earlier containers' sizes
   (fewer than 4), and more than 65 535 expand items in one call.
B. sorted columns: docId-range leaves (PB_F_SORTED) and the bit-packed stream pb_sorted_to_packed_kernel writes for group
   keys and aggregation inputs.
C. chunk-compressed raw forward indexes (pb_chunk_decode_kernel): LZ4, LZ4_LENGTH_PREFIXED and SNAPPY streams with chosen
   stream features (the encoders below), pyarrow's stock compressors, writer versions 1 to 4, and malformed chunks.

Every segment carries blk = doc >> 5 (a dictionary INT column) and did (a raw LONG, a random 40-bit value per doc).  The
filter queries group by blk with COUNT(*), SUM / MIN / MAX of did: that names the admitted docs of every 32-doc word of
the flat doc bitmap, so one wrong bit fails the comparison.  A group holds at most 32 docs per segment, so its sums stay
far below 2^53 and compare exactly.  The CPU tests check that the data reaches the edges it is built for, so a change to
the writer cannot quietly shrink what the device tests cover."""
import contextlib
import functools

import numpy as np
import pytest

from pinot_b200 import native
from pinot_b200.query import parse_sql
from pinot_b200.segment_writer import DataType, build_column, build_dict_column, make_segment, with_nulls
from tests.parity import check_query
from tests.reference import Col
from tests.test_cpu_formats import _roaring_decode_py
from tests.test_gpu_fuzz import FLAGS, run_and_check

C64 = 65536
NGL = "SET numGroupsLimit = 100000000; "
FP = ("COUNT(*)", "SUM(did)", "MIN(did)", "MAX(did)")


def _fp_sql(where):
    return f"{NGL}SELECT blk, {', '.join(FP)} FROM t WHERE {where} GROUP BY blk LIMIT 100000000"


def _fp_filter_sql(clauses):
    """the fingerprint of each clause as a FILTER(WHERE ...) swim-lane (at most 3 clauses: 16 aggregations)"""
    aggs = ", ".join(f"{a} FILTER(WHERE {c})" for c in clauses for a in FP)
    return f"{NGL}SELECT blk, COUNT(*), {aggs} FROM t GROUP BY blk LIMIT 100000000"


def _base(n, rng):
    blk = np.arange(n, dtype=np.int64) >> 5
    did = rng.integers(0, 2 ** 40, n).astype(np.int64)
    cols = [build_column("blk", DataType.INT, blk.astype(np.int32)), build_column("did", DataType.LONG, did, dictionary=False)]
    return cols, {"blk": Col(blk, DataType.INT), "did": Col(did, DataType.LONG, False)}


def _dict_col(name, values, ids, run_optimize=True):
    """an inverted INT column over the dictionary `values`; a column whose ids happen to be sorted (a tiny segment) is
    written as a sorted column with only the entries it uses"""
    ids = np.asarray(ids, np.int64)
    if ids.size <= 1 or (ids[1:] >= ids[:-1]).all():
        used, ids = np.unique(ids, return_inverse=True)
        values = values[used]
    return build_dict_column(name, DataType.INT, values, ids.astype(np.uint32), inverted=True, run_optimize=run_optimize)


@contextlib.contextmanager
def _group(segs):
    staged = [native.StagedSegment(s) for s in segs]
    g = native.SegmentGroup(staged)
    try:
        yield g
    finally:
        g.release()
        for s in staged:
            s.release()


@pytest.fixture(scope="module")
def device():
    native.init()


# ==== A. Roaring containers: inverted-index leaves and null-value vectors ====

A_SIZES = (1, 31, 32, 33, 65_535, 65_536, 65_537, 200_003, 330_017)
N_IDS = 50                       # dictIds per shaped column: the designed doc sets, the other docs spread over the rest
VALS = np.arange(N_IDS, dtype=np.int64) * 7 - 100
INT_NULL = -(2 ** 31)            # the default null value of an INT dimension


class _Layout:
    """dictIds of n docs, set shape by shape (doc sets of one id may not overlap another's); positions are (container,
    offset in the container) and are clipped to the segment"""

    def __init__(self, n, rng):
        self.n, self.rng, self.ids = n, rng, np.full(n, -1, np.int64)

    def put(self, d, docs):
        docs = np.asarray(docs, np.int64)
        docs = docs[docs < self.n]
        assert (self.ids[docs] == -1).all()
        self.ids[docs] = d

    def run(self, d, c, lo, hi):                     # docs [lo, hi) of container c
        self.put(d, c * C64 + np.arange(lo, hi))

    def some(self, d, c, lo, hi, k):                 # k random docs of [lo, hi) of container c
        self.put(d, c * C64 + np.sort(self.rng.choice(np.arange(lo, hi), k, replace=False)))

    def fill(self, designed):
        free = self.ids < 0
        others = np.array([i for i in range(N_IDS) if i not in designed])
        self.ids[free] = self.rng.choice(others, int(free.sum()))
        return self.ids


KC_IDS = list(range(1, 10))
KE_IDS = list(range(1, 8))


def _kc(L):
    """container counts and the kinds the walk steps over (kinds under run_optimize; without it every run is an array or
    a bitmap container)"""
    L.put(1, np.arange(0, 8192, 2)); L.put(1, C64 + np.arange(0, 8194, 2))                    # 4096 docs: array, 4097: bitmap
    L.run(2, 0, 10000, 20000); L.some(2, 1, 10000, 40000, 5000); L.some(2, 2, 0, 5000, 100)   # run, bitmap, array
    L.some(3, 0, 30000, 40000, 50); L.run(3, 1, 50000, 60001); L.some(3, 2, 10000, 30000, 6000)   # array, run, bitmap
    L.some(9, 0, 20000, 30000, 6000); L.some(9, 1, 40000, 45000, 40); L.run(9, 2, 61500, 62500)   # bitmap, array, run
    L.run(4, 0, 45000, 46000); L.some(4, 1, 45000, 45600, 300); L.some(4, 2, 30000, 50000, 5000); L.run(4, 3, 0, 3000)
    L.some(5, 0, 58000, 60000, 20); L.run(5, 1, 62500, 63500); L.some(5, 2, 50000, 60000, 5000)
    L.some(5, 3, 10000, 12000, 30); L.run(5, 4, 0, 20000)                                       # 5 containers
    L.run(6, 0, 50000, 50011)                                                                   # 1 container
    L.run(7, 0, 52000, 53000); L.some(7, 1, 61000, 62000, 100)                                  # 2: run, array
    L.some(8, 0, 55000, 58000, 200); L.run(8, 2, 60000, 61000); L.some(8, 5, 0, 2337, 500)      # keys 0, 2, 5 (partial)
    return L.fill(KC_IDS)


def _ke(L):
    """run edges and the run / plain choice (the writer takes the run form when it is smaller; sizes are even, so one
    step is 2 bytes)"""
    for lo, hi in ((320, 352), (671, 673), (967, 968), (1311, 1312), (1600, 1601), (1923, 9618)):
        L.put(1, np.arange(lo, hi))          # bits 0-31 of a word, bit 31 into bit 0 of the next, single docs at bits 7, 31, 0
    L.put(2, [*range(10000, 10007), 10010, 10020, 10030])          # 10 docs in 4 runs: run 18 bytes < array 20
    L.put(3, [11000 + 10 * k + j for k in range(5) for j in range(2)])   # 10 docs in 5 runs: run 22 > array 20
    L.put(4, 20000 + (np.arange(2047)[:, None] * 4 + np.arange(3)).ravel())   # 2047 runs: 8190 < bitmap 8192
    L.put(5, 30000 + (np.arange(2048)[:, None] * 4 + np.arange(3)).ravel())   # 2048 runs: 8194 > 8192
    L.run(6, 1, 0, C64)                                                          # all 65 536 docs of a container
    L.run(7, 2, C64 - 1000, C64); L.run(7, 3, 0, 1000)                          # one run across two containers
    return L.fill(KE_IDS)


NULL_COLS = ("nall", "nfirst", "nalt", "nsparse")


@functools.lru_cache(maxsize=None)
def a_table():
    segs, srcs = [], []
    for si, n in enumerate(A_SIZES):
        rng = np.random.default_rng(4200 + si)
        cols, src = _base(n, rng)
        for name, design in (("kc", _kc), ("ke", _ke)):
            ids = design(_Layout(n, rng))
            for ro in (True, False):
                cols.append(_dict_col(f"{name}_{'r' if ro else 'p'}", VALS, ids, ro))
                src[f"{name}_{'r' if ro else 'p'}"] = Col(VALS[ids], DataType.INT)
        doc = np.arange(n)
        for name, nulls in zip(NULL_COLS, (np.ones(n, bool), doc < 100_000, doc % 2 == 1, rng.random(n) < 0.005)):
            v = np.where(nulls, INT_NULL, rng.integers(0, 20, n)).astype(np.int64)
            cols.append(with_nulls(build_column(name, DataType.INT, v.astype(np.int32)), nulls))
            src[name] = Col(v, DataType.INT, True, nulls)
        segs.append(make_segment(f"roaring{si}", cols))
        srcs.append(src)
    return segs, srcs


def cards_all(lays, kind):
    return {c for l in lays for _, c, k in l["containers"] if k == kind}


def _blobs(col):
    """(dictId, blob) of every bitmap of an inverted index"""
    inv = col.inverted_index.tobytes()
    offs = np.frombuffer(inv[:4 * (col.cardinality + 1)], ">u4").astype(np.int64)
    return [(d, inv[offs[d]:offs[d + 1]]) for d in range(col.cardinality)]


def test_roaring_blobs_reach_every_container_edge():
    """The designed columns decode to the designed doc sets, and the blobs hold every layout pb_expand_kernel reads."""
    segs, srcs = a_table()
    seen = []                        # (segment size, column, dictId, layout)
    for seg, src in zip(segs, srcs):
        for name in ("kc_r", "kc_p", "ke_r", "ke_p"):
            c = seg.columns[name]
            if c.is_sorted:
                continue
            vals = src[name].values
            for d, blob in _blobs(c):
                lay = {}
                assert _roaring_decode_py(blob, lay) == np.flatnonzero(vals == VALS[d]).tolist(), (seg.num_docs, name, d)
                seen.append((seg.num_docs, name, d, lay))
        for name in NULL_COLS:
            v = seg.columns[name].null_value_vector
            if v is not None:
                lay = {}
                assert _roaring_decode_py(v.tobytes(), lay) == np.flatnonzero(src[name].nulls).tolist()
                seen.append((seg.num_docs, name, -1, lay))

    def kinds(lay):
        return [k for _, _, k in lay["containers"]]

    lays = [s[3] for s in seen]
    assert any(l["cookie"] == 12346 for l in lays)
    assert any(l["cookie"] == 12347 and l["offsets"] for l in lays)
    assert {"array", "bitmap", "run"} <= {k for l in lays for k in kinds(l)}
    walks = {tuple(kinds(l)) for l in lays if l["cookie"] == 12347 and not l["offsets"]}
    for shape in (("run",), ("run", "array"), ("run", "bitmap", "array"), ("array", "run", "bitmap"), ("bitmap", "array", "run")):
        assert shape in walks, shape                       # the walk steps over each kind before the container it reads
    counts = {len(l["containers"]) for l in lays if l["cookie"] == 12347}
    assert {1, 2, 3, 4, 5} <= counts
    assert 4096 in cards_all(lays, "array") and 4097 in cards_all(lays, "bitmap")
    assert C64 in cards_all(lays, "run")                   # one run of a whole container
    assert 10 in cards_all(lays, "run") and 10 in cards_all(lays, "array")   # the run / array choice on either side
    assert 6141 in cards_all(lays, "run") and 6144 in cards_all(lays, "bitmap")   # the run / bitmap choice
    assert any(kinds(l) == ["run", "run"] for (_, name, d, l) in seen if name == "ke_r" and d == 7)   # a run across containers
    assert any([k for k, _, _ in l["containers"]] == [0, 2, 5] for l in lays)                        # key gaps
    big = max(A_SIZES)
    assert any(l["containers"][-1][0] == (big - 1) >> 16 for (n, _, _, l) in seen if n == big)      # a partial last container
    # the null-value vectors: runs (every doc null, the first 100 000 null), bitmaps (alternating docs), arrays (sparse)
    nv = {name: set(k for (n, nm, _, l) in seen if nm == name and n == big for k in kinds(l)) for name in NULL_COLS}
    assert nv["nall"] == {"run"} and "run" in nv["nfirst"] and "bitmap" in nv["nalt"] and nv["nsparse"] == {"array"}


def _lit(ids):
    return ", ".join(str(int(VALS[d])) for d in ids)


def _a_queries(col, designed):
    """the leaf forms over the designed dictIds; per dictId (FILTER swim-lanes) where the blobs hold run containers"""
    s = designed
    return [_fp_sql(f"{col} IN ({_lit(s)})"), _fp_sql(f"{col} NOT IN ({_lit(s)})"), _fp_sql(f"{col} <> {_lit([s[1]])}"),
            _fp_sql(f"{col} = {_lit([s[-1]])}"), _fp_sql(f"NOT ({col} IN ({_lit(s[::2])}))"),
            _fp_sql(f"{col} IN ({_lit(s[1::2])}) OR did < {2 ** 35}"),
            # an index leaf that keeps 2 % of the docs ahead of a scan leaf: the scan leaf runs on its candidates
            _fp_sql(f"{col} = {_lit([s[2]])} AND did < {2 ** 39}")] + \
        [_fp_filter_sql([f"{col} = {_lit([d])}" for d in s[i:i + 3]]) for i in range(0, len(s), 3) if col.endswith("_r")]


@pytest.mark.gpu
@pytest.mark.parametrize("col", ["kc_r", "kc_p", "ke_r", "ke_p"])
def test_inverted_leaves_over_every_container_layout(device, col):
    segs, srcs = a_table()
    designed = KC_IDS if col.startswith("kc") else KE_IDS
    with _group(segs) as g:
        lowered = native.dump_lowered(g, parse_sql(_fp_sql(f"{col} IN ({_lit(designed)})")), segment_index=len(segs) - 1)
        assert any(line.startswith("INVERTED") for line in lowered), lowered
        for sql in _a_queries(col, designed):
            run_and_check(g, segs, srcs, sql, f"roaring {col}")
        res = native.execute(g, parse_sql(_fp_sql(f"{col} = {_lit([designed[2]])} AND did < {2 ** 39}")), native.PB_Q_COMBINE)
        assert res.plan_info["cand_leaf"] > 0, res.plan_info
        res.free()


@pytest.mark.gpu
def test_is_null_over_null_value_vectors(device):
    segs, srcs = a_table()
    with _group(segs) as g:
        for sql in (_fp_sql("nall IS NULL"), _fp_sql("nfirst IS NOT NULL"), _fp_sql("NOT (nalt IS NULL)"),
                    _fp_sql("nsparse IS NULL"), _fp_sql(f"nsparse IS NULL OR did < {2 ** 35}"),
                    _fp_sql(f"nfirst IS NULL AND nalt IS NOT NULL AND did < {2 ** 39}"),
                    _fp_filter_sql(["nfirst IS NULL", "nalt IS NOT NULL", "NOT (nsparse IS NULL)"]),
                    _fp_filter_sql(["nall IS NOT NULL", "nsparse IS NOT NULL", "nalt IS NULL AND kc_r <> -93"])):
            run_and_check(g, segs, srcs, sql, "nulls")
        check_query(segs, "SET enableNullHandling=true; " + NGL + "SELECT blk, COUNT(*), COUNT(nfirst), SUM(nfirst), MIN(nfirst), "
                    "MAX(nfirst) FROM t WHERE nfirst > 3 OR blk < 100 GROUP BY blk LIMIT 100000000", group=g, flags_list=FLAGS)


@functools.lru_cache(maxsize=None)
def wide_in_table():
    """three segments whose inverted column has 32 768 dictIds, for an IN list of 30 000 of them"""
    segs, srcs = [], []
    vals = np.arange(32_768, dtype=np.int64) * 3 + 1
    for si in range(3):
        rng = np.random.default_rng(4300 + si)
        n = 40_000 + 17 * si
        cols, src = _base(n, rng)
        ids = rng.integers(0, vals.size, n)
        cols.append(build_dict_column("w", DataType.INT, vals, ids.astype(np.uint32), inverted=True))
        src["w"] = Col(vals[ids], DataType.INT)
        segs.append(make_segment(f"wide{si}", cols))
        srcs.append(src)
    in_list = ", ".join(str(int(v)) for v in vals[np.random.default_rng(4399).choice(vals.size, 30_000, replace=False)])
    return segs, srcs, in_list


def test_wide_in_list_lowers_to_more_than_65535_expand_items():
    """one expand item per (segment, dictId) of an inverted leaf: the y-chunked launch loop of pb_expand_kernel runs"""
    segs, srcs, in_list = wide_in_table()
    with _group(segs) as g:
        for op in ("IN", "NOT IN"):
            q = parse_sql(_fp_sql(f"w {op} ({in_list})"))
            items = 0
            for si in range(len(segs)):
                inv = [line for line in native.dump_lowered(g, q, segment_index=si) if line.startswith("INVERTED")]
                assert len(inv) == 1, inv
                items += len(inv[0].split("ids=")[1].split(","))
            assert items == 90_000 > 65_535


@pytest.mark.gpu
def test_more_than_65535_expand_items(device):
    segs, srcs, in_list = wide_in_table()
    with _group(segs) as g:
        for op in ("IN", "NOT IN"):
            run_and_check(g, segs, srcs, _fp_sql(f"w {op} ({in_list})"), f"wide {op}")


# ==== B. sorted columns ====

B_SIZES = (1, 33, 4_099, 70_001)
B_CARDS = (1, 2, 3, 16, 17, 128, 129, 4096, 4097)


def _sorted_ids(n, card, rng):
    """dictIds 0..card-1 in runs: single-doc runs at the start, runs that end on bit 31 of a word, a final run of one doc"""
    card = min(card, n)
    forced = [b for b in (n - 1, 32, 1, 2, 64, 96, 127, 128) if 0 < b < n]
    starts = list(dict.fromkeys(forced))[:card - 1]
    rest = np.setdiff1d(np.arange(1, n), starts)
    starts = np.sort(np.concatenate([starts, rng.choice(rest, card - 1 - len(starts), replace=False)])).astype(np.int64)
    return np.searchsorted(starts, np.arange(n), side="right")


@functools.lru_cache(maxsize=None)
def b_table():
    segs, srcs = [], []
    for si, n in enumerate(B_SIZES):
        rng = np.random.default_rng(4400 + si)
        cols, src = _base(n, rng)
        for card in B_CARDS:
            ids = _sorted_ids(n, card, rng)
            vals = np.arange(ids.max() + 1, dtype=np.int64) * 3 - 7
            cols.append(build_dict_column(f"s{card}", DataType.INT, vals, ids.astype(np.uint32)))
            src[f"s{card}"] = Col(vals[ids], DataType.INT)
        segs.append(make_segment(f"sorted{si}", cols))
        srcs.append(src)
    return segs, srcs


def test_sorted_columns_reach_their_edges():
    segs, _ = b_table()
    big = segs[-1]
    assert all(c.is_sorted for c in big.columns.values() if c.name.startswith("s"))
    assert [big.columns[f"s{c}"].bits_per_element for c in B_CARDS] == [1, 1, 2, 4, 5, 7, 8, 12, 13]   # 5, 7, 13 straddle words
    for seg in segs:
        assert seg.num_docs % 32
        for card in B_CARDS:
            c = seg.columns[f"s{card}"]
            pairs = np.frombuffer(c.forward_index.tobytes(), ">i4").reshape(-1, 2)
            if c.cardinality > 1:
                assert pairs[-1, 0] == pairs[-1, 1] == seg.num_docs - 1                    # a final run of one doc
            if c.cardinality > 2:
                assert (pairs[:-1, 1] % 32 == 31).any()                                    # a run ending on bit 31
            if c.cardinality > 3:
                assert pairs[0, 0] == pairs[0, 1] == 0                                     # a run of one doc


def _s(card, k):
    return int(k) * 3 - 7


B_LEAF_COLS = (3, 17, 129, 4097)


@pytest.mark.gpu
def test_sorted_leaves_keys_and_inputs(device):
    segs, srcs = b_table()
    sqls = []
    for card in B_LEAF_COLS:
        c, hi = f"s{card}", card - 1
        clauses = [f"{c} = {_s(card, hi // 2)}", f"{c} IN ({_s(card, 0)}, {_s(card, 1)}, {_s(card, hi // 3)}, {_s(card, hi)})",
                   f"{c} BETWEEN {_s(card, 1)} AND {_s(card, hi - 1)}", f"{c} <> {_s(card, hi)}",
                   f"{c} NOT IN ({_s(card, 0)}, {_s(card, hi // 2)}, {_s(card, hi)})"]
        sqls += [_fp_sql(clauses[0]), _fp_sql(clauses[4]), _fp_filter_sql(clauses[:3]), _fp_filter_sql(clauses[3:])]
    sqls += [f"{NGL}SELECT blk, SUM(s17), MIN(s129), MAX(s4097), SUM(s4097), SUM(s3), SUM(s2), SUM(s1), SUM(s128), SUM(s4096), "
             "SUM(s16) FROM t GROUP BY blk LIMIT 100000000",
             f"{NGL}SELECT blk, DISTINCTCOUNT(s4097), DISTINCTCOUNT(s129), DISTINCTCOUNT(s17) FROM t GROUP BY blk LIMIT 100000000",
             f"{NGL}SELECT s4097, COUNT(*), SUM(did), MIN(did), MAX(did) FROM t GROUP BY s4097 LIMIT 100000000",
             f"{NGL}SELECT s129, s17, s3, s1, COUNT(*), SUM(did), MAX(did) FROM t WHERE s2 = {_s(2, 1)} GROUP BY s129, s17, s3, s1 LIMIT 100000000",
             f"{NGL}SELECT s16, s2, COUNT(*), DISTINCTCOUNT(s128), SUM(s4096) FROM t GROUP BY s16, s2 LIMIT 100000000"]
    with _group(segs) as g:
        for sql in sqls:
            run_and_check(g, segs, srcs, sql, "sorted")


# ==== C. chunk codecs ====
# A stream is written from a script of ("lit", bytes[, extra length bytes]) and ("copy", offset, length) items; _play
# executes a script the way the format defines (a copy may overlap its own output), and the encoders write it as an LZ4
# block or a Snappy stream and report the element kinds they emitted.

def _play(items) -> bytes:
    out = bytearray()
    for it in items:
        if it[0] == "lit":
            out += it[1]
        else:
            off, n = it[1], it[2]
            assert 1 <= off <= len(out)
            pat = bytes(out[len(out) - off:])
            out += (pat * (n // off + 1))[:n]
    return bytes(out)


def _lz4_len(n):
    b = bytearray()
    n -= 15
    while n >= 255:
        b.append(255)
        n -= 255
    b.append(n)
    return b


def lz4_block(items):
    """LZ4 block of a script: every copy (length >= 4) closes a sequence with the literals before it; the script ends in
    at least 12 literal bytes (liblz4's end-of-block rules: the last 5 bytes are literals, the last match starts 12 or
    more bytes before the end).  Returns (block, kinds)."""
    out, kinds, lits = bytearray(), set(), bytearray()
    for it in items + [("end",)]:
        if it[0] == "lit":
            lits += it[1]
            continue
        ml = None if it[0] == "end" else it[2] - 4
        ln = len(lits)
        out.append((min(ln, 15) << 4) | (0 if ml is None else min(ml, 15)))
        if ln >= 15:
            out += _lz4_len(ln)
        out += lits
        kinds.add(("lz4 literal length", ln))
        lits = bytearray()
        if ml is None:
            assert ln >= 12 or len(out) == ln + 1 + (ln >= 15)      # (a block of literals alone may be short)
            break
        assert ml >= 0 and 1 <= it[1] <= 65535
        out += it[1].to_bytes(2, "little")
        if ml >= 15:
            out += _lz4_len(ml)
        kinds |= {("lz4 match length", ml), ("offset", it[1])}
        if it[1] < it[2] and it[2] > 32:
            kinds.add(("overlapping copy", it[1]))
    return bytes(out), kinds


def _varint(n):
    b = bytearray()
    while n >= 128:
        b.append(n & 127 | 128)
        n >>= 7
    b.append(n)
    return b


def snappy_stream(items, total=None):
    """Snappy stream of a script: the preamble (total, default the decoded length), literals with 0-4 length bytes (the
    item's third field forces a longer encoding), copies as copy-1 (length 4-11, offset < 2048), copy-2 (offset < 65536)
    or copy-4, in pieces of at most 64 bytes.  Returns (stream, kinds)."""
    out, kinds = bytearray(_varint(len(_play(items)) if total is None else total)), set()
    for it in items:
        if it[0] == "lit":
            n1 = len(it[1]) - 1
            nb = it[2] if len(it) > 2 else (0 if n1 < 60 else (n1.bit_length() + 7) // 8)
            out += bytes([n1 << 2]) if nb == 0 else bytes([(59 + nb) << 2]) + n1.to_bytes(nb, "little")
            out += it[1]
            kinds |= {("snappy literal length bytes", nb), ("snappy literal", len(it[1]), nb)}
            continue
        off, n = it[1], it[2]
        form = it[3] if len(it) > 3 else None
        while n > 0:
            k = min(n, 64 if form != 1 else 11)
            f = form or (1 if 4 <= k <= 11 and off < 2048 else 2 if off < 65536 else 4)
            if f == 1:
                assert 4 <= k <= 11 and off < 2048
                out += bytes([(off >> 8) << 5 | (k - 4) << 2 | 1, off & 255])
            else:
                out += bytes([(k - 1) << 2 | (2 if f == 2 else 3)]) + off.to_bytes(2 if f == 2 else 4, "little")
            kinds.add((f"copy-{f}", off))
            if off < k and k > 32:
                kinds.add(("overlapping copy", off))
            n -= k
    return bytes(out), kinds


def greedy_script(data: bytes, min_off=1, max_off=65535):
    """a greedy matcher over data: the latest earlier position with the same 4 bytes, taken when its offset is in
    [min_off, max_off]; the last 12 bytes stay literals"""
    items, last, i, lit0, end = [], {}, 0, 0, len(data) - 12
    while i < end:
        key = data[i:i + 4]
        j = last.get(key)
        last[key] = i
        if j is not None and min_off <= i - j <= max_off:
            n = 0
            while i + n < end and data[j + n] == data[i + n]:
                n += 1
            if n >= 4:
                if i > lit0:
                    items.append(("lit", data[lit0:i]))
                items.append(("copy", i - j, n))
                i += n
                lit0 = i
                continue
        i += 1
    items.append(("lit", data[lit0:]))
    return items


OVERLAP_OFFSETS = (1, 2, 3, 7, 8, 31, 32, 33)
LZ4_FIELDS = (14, 15, 15 + 254, 15 + 255, 15 + 600)      # literal and match-length fields: 0, 1 (=0), 1, 2 (255, 0), 3 bytes
SNAPPY_LITERALS = ((60, 0), (61, 1), (256, 1), (257, 2), (65_536, 2), (65_537, 3))


def _feature_script(rng, size, codec, part):
    """one chunk of `size` bytes: the stream features of `codec` that fit (part 0 and 1 split the long Snappy literals over
    two chunks), then random literals and copies, then 12 or more closing literals"""
    items, op = [], 0

    def lit(n, nb=None):
        nonlocal op
        items.append(("lit", rng.integers(0, 256, n, dtype=np.uint8).tobytes()) + (() if nb is None else (nb,)))
        op += n

    def copy(off, n, form=None):
        nonlocal op
        items.append(("copy", off, n) + (() if form is None else (form,)))
        op += n

    room = lambda n: op + n + 400 <= size
    if codec == "lz4":
        lit(14)
        for k, off in enumerate(OVERLAP_OFFSETS):
            copy(off, 40 + 3 * k)
            lit(LZ4_FIELDS[k % len(LZ4_FIELDS)])
        for f in LZ4_FIELDS:
            copy(int(rng.integers(1, op)), f + 4)
            lit(int(rng.integers(1, 9)))
        if room(C64):
            lit(C64)
            copy(65_535, 40)
    else:
        lit(40)
        for off in OVERLAP_OFFSETS:
            copy(off, 40 + off, 2)
        for n, nb in SNAPPY_LITERALS[:4] + (SNAPPY_LITERALS[4 + part:5 + part] if part < 2 else ()):
            if room(n):
                lit(n)
        lit(5, 4)                                                   # a 5-byte literal with a 4-byte length
        if op < 2047:
            lit(2100)
        copy(2047, 8, 1)
        if op > 65_535:
            copy(65_535, 50, 2)
        copy(int(rng.integers(1, op)), 60, 4)
        copy(300, 64, 4)
    while size - op >= 400:
        lit(int(rng.integers(1, 20)))
        copy(int(rng.integers(1, min(op, 65_535) + 1)), int(rng.integers(4, 300)))
    lit(size - op)
    assert len(_play(items)) == size
    return items


C_SIZES = (32_769, 16_385)           # every power-of-two chunk leaves a last chunk of one doc
C_NAMES = {"LZ4": "zlz", "LZ4_LENGTH_PREFIXED": "zlp", "SNAPPY": "zsn"}
C_LAYOUTS = [(comp, v, 16_384 if v != 3 else 4_096) for comp in ("LZ4", "LZ4_LENGTH_PREFIXED", "SNAPPY") for v in (2, 3, 4)] + \
    [("SNAPPY", 1, 16_384)]


def _encode(comp, items):
    return (snappy_stream if comp == "SNAPPY" else lz4_block)(items)


@functools.lru_cache(maxsize=None)
def c_table():
    """(segments, sources, {column: [(codec, script, stream, kinds) per chunk]})"""
    segs, srcs, streams = [], [], {}
    for si, n in enumerate(C_SIZES):
        rng = np.random.default_rng(4500 + si)
        cols, src = _base(n, rng)

        def add(name, dt, vals, comp, version, dpc, block=None):
            cols.append(build_column(name, dt, vals, dictionary=False, raw_compression=comp, raw_version=version,
                                     raw_docs_per_chunk=dpc, raw_block=block))
            cols.append(build_column("p" + name, dt, vals, dictionary=False))
            for nm in (name, "p" + name):
                src[nm] = Col(np.asarray(vals).astype(np.float64 if dt == DataType.DOUBLE else np.int64), dt, False)

        def scripted(name, comp, version, dpc, make):
            chunks, raw = [], []
            for k in range(-(-n // dpc)):
                size = 8 * min(dpc, n - k * dpc)
                items = make(k, size)
                stream, kinds = _encode(comp, items)
                chunks.append((comp, items, stream, kinds))
                raw.append(_play(items))
            table = {r: s for r, (_, _, s, _) in zip(raw, chunks)}
            vals = np.frombuffer(b"".join(raw), ">i8").astype(np.int64)
            add(name, DataType.LONG, vals, comp, version, dpc, table.__getitem__)
            streams[(si, name)] = chunks
        for comp, version, dpc in C_LAYOUTS:
            codec = "snappy" if comp == "SNAPPY" else "lz4"
            scripted(f"{C_NAMES[comp]}{version}", comp, version, dpc,
                     lambda k, size: _feature_script(rng, size, codec, k) if size > 8 else [("lit", rng.bytes(8))])
        small = np.where(rng.random(n) < 0.1, rng.integers(0, 8, n), 0).astype(np.int64)   # long runs of zero bytes
        for comp, lo, hi in (("LZ4", 9, 65_535), ("SNAPPY", 1, 2047)):
            scripted(f"g{comp.lower()}", comp, 2, 4096,
                     lambda k, size: greedy_script((small[k * 4096:k * 4096 + size // 8] * 977).astype(">i8").tobytes(), lo, hi))
        # pyarrow's compressors on the shapes real columns take
        add("const", DataType.INT, np.full(n, 7, np.int32), "LZ4", 3, 1000)
        add("smalli", DataType.INT, small.astype(np.int32), "SNAPPY", 2, 4096)
        add("incr", DataType.LONG, np.cumsum(rng.integers(-2, 40, n)).astype(np.int64), "LZ4_LENGTH_PREFIXED", 4, 16_384)
        add("dbl", DataType.DOUBLE, rng.normal(0, 1e3, n), "SNAPPY", 3, 1000)
        segs.append(make_segment(f"codec{si}", cols))
        srcs.append(src)
    return segs, srcs, streams


def test_encoders_round_trip_and_emit_every_stream_feature():
    """Every stream the encoders emit for the device tests decodes, through pyarrow's liblz4 / libsnappy and through the
    oracle, to the bytes its script plays; together the streams hold every feature the device tests aim at."""
    pa = pytest.importorskip("pyarrow")
    from oracle import oracle
    _, _, streams = c_table()
    kinds = set()
    for (si, name), chunks in streams.items():
        for comp, items, stream, k in chunks:
            raw = _play(items)
            codec = "snappy" if comp == "SNAPPY" else "lz4"
            assert pa.Codec("snappy" if codec == "snappy" else "lz4_raw").decompress(stream, len(raw), asbytes=True) == raw, name
            assert oracle.block_decode(codec, stream, len(raw)) == raw, name
            kinds |= {(codec,) + x for x in k}
    for off in OVERLAP_OFFSETS:
        assert ("lz4", "overlapping copy", off) in kinds and ("snappy", "overlapping copy", off) in kinds, off
    for f in LZ4_FIELDS:
        assert ("lz4", "lz4 literal length", f) in kinds and ("lz4", "lz4 match length", f) in kinds, f
    assert ("lz4", "offset", 65_535) in kinds
    for n, nb in SNAPPY_LITERALS + ((5, 4),):
        assert ("snappy", "snappy literal", n, nb) in kinds, (n, nb)
    assert {("snappy", "copy-1", 2047), ("snappy", "copy-2", 65_535)} <= kinds
    assert any(k[:2] == ("snappy", "copy-4") for k in kinds)
    assert any(k[:2] == ("lz4", "offset") and k[2] > 8 for k in kinds)


def test_writer_versions_and_chunk_sizes():
    """writer versions 1 (four header ints, int offsets, SNAPPY implied) to 4; chunks over 64 KiB; a last chunk of one
    doc; the oracle reads each index back as the plain values"""
    import struct
    from oracle import oracle
    segs, srcs, _ = c_table()
    for seg, src in zip(segs, srcs):
        for comp, version, dpc in C_LAYOUTS:
            name = f"{C_NAMES[comp]}{version}"
            raw = seg.columns[name].forward_index.tobytes()
            head = struct.unpack_from(">4i", raw, 0)
            assert head == (version, -(-seg.num_docs // dpc), dpc, 8) and seg.num_docs % dpc == 1
            first = struct.unpack_from(">i" if version <= 2 else ">q", raw, 16 if version == 1 else 28)[0]
            assert first == (16 if version == 1 else 28) + head[1] * (4 if version <= 2 else 8)
            assert dpc * 8 > C64 or version == 3
            back = oracle.raw_forward_decompress(seg.columns[name].forward_index, 8, seg.num_docs)
            assert (np.frombuffer(back.tobytes()[-8 * seg.num_docs:], ">i8") == src[name].values).all()


C_COLS = [f"{C_NAMES[comp]}{v}" for comp, v, _ in C_LAYOUTS] + ["glz4", "gsnappy", "const", "smalli", "incr", "dbl"]


@pytest.mark.gpu
def test_chunk_codecs_against_the_reference_and_a_plain_twin(device):
    """each compressed column as a filter leaf and SUM / MIN / MAX input next to its PASS_THROUGH twin (same values, same
    segment); the small-range INT columns also as group keys"""
    segs, srcs, _ = c_table()
    with _group(segs) as g:
        for c in C_COLS:
            v = np.concatenate([s[c].values for s in srcs])
            cut = np.median(v)
            cut = repr(float(cut)) if c == "dbl" else str(int(cut))
            sql = f"{NGL}SELECT blk, COUNT(*), SUM({c}), MIN({c}), MAX({c}), SUM(p{c}), MIN(p{c}), MAX(p{c}) FROM t " \
                  f"WHERE {c} >= {cut} GROUP BY blk LIMIT 100000000"
            run_and_check(g, segs, srcs, sql, f"codec {c}")
            res = native.execute(g, parse_sql(sql), native.PB_Q_COMBINE)
            for key, row in res.tables[0].rows().items():
                assert row[2:4] == row[5:7], f"{c} {key}: {row}"        # MIN / MAX of the column and of its twin
            res.free()
            twin = f"{NGL}SELECT blk, {', '.join(FP)} FROM t WHERE p{c} >= {cut} GROUP BY blk LIMIT 100000000"
            run_and_check(g, segs, srcs, twin, f"codec twin p{c}")
        run_and_check(g, segs, srcs, f"{NGL}SELECT smalli, const, {', '.join(FP)}, SUM(incr) FROM t WHERE incr > 1000 "
                      "GROUP BY smalli, const LIMIT 100000000", "codec keys")


def _malformed(case, raw):
    """chunk 0 of a column rewritten as a stream the decoder must refuse; raw = its true bytes"""
    pa = pytest.importorskip("pyarrow")
    body = [("lit", raw[:16]), ("copy", 8, len(raw) - 28), ("lit", raw[-12:])]
    if case == "lz4 offset past the output":
        return lz4_block([("lit", raw[:4]), ("copy", 5, 20), ("lit", raw[-12:])])[0]
    if case == "lz4 match past the chunk":
        return lz4_block([("lit", raw[:16]), ("copy", 8, len(raw)), ("lit", raw[-12:])])[0]
    if case == "lz4 literals past the input":
        return lz4_block([("lit", raw)])[0][:len(raw) // 2]
    if case == "snappy offset past the output":
        return snappy_stream([("lit", raw[:4]), ("copy", 5, 20), ("lit", raw[24:])], len(raw))[0]
    if case == "snappy preamble":
        return snappy_stream([("lit", raw)], len(raw) + 8)[0]
    if case == "lz4 prefix":
        return (len(raw) - 8).to_bytes(4, "little") + pa.Codec("lz4_raw").compress(raw, asbytes=True)
    if case == "lz4 one byte short":
        return lz4_block(body)[0][:-1]
    if case == "snappy one byte short":
        return snappy_stream(body)[0][:-1]
    if case == "lz4 decodes short":
        return lz4_block([("lit", raw[:-8])])[0]
    assert case == "snappy decodes short"
    return snappy_stream([("lit", raw[:-8])], len(raw))[0]


PB_ERR_INVALID = -1                  # include/pinot_b200.h
MALFORMED = ["lz4 offset past the output", "lz4 match past the chunk", "lz4 literals past the input", "snappy offset past the output",
             "snappy preamble", "lz4 prefix", "lz4 one byte short", "snappy one byte short", "lz4 decodes short", "snappy decodes short"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", MALFORMED)
def test_malformed_chunk_is_rejected(device, case):
    """The first of five chunks is malformed, so a decoder without its bounds check would still read inside the staged
    buffer and write inside the value area: the call fails with PB_ERR_INVALID and no result."""
    import pyarrow as pa
    rng = np.random.default_rng(4600)
    n, dpc = 5000, 1000
    vals = np.cumsum(rng.integers(0, 5, n)).astype(np.int64)
    raw0 = vals[:dpc].astype(">i8").tobytes()
    comp = "SNAPPY" if case.startswith("snappy") else "LZ4_LENGTH_PREFIXED" if case == "lz4 prefix" else "LZ4"
    bad = _malformed(case, raw0)

    def block(raw):
        if raw == raw0:
            return bad[4:] if comp == "LZ4_LENGTH_PREFIXED" else bad
        return pa.Codec("snappy" if comp == "SNAPPY" else "lz4_raw").compress(raw, asbytes=True)
    cols, _ = _base(n, rng)
    col = build_column("k", DataType.LONG, vals, dictionary=False, raw_compression=comp, raw_docs_per_chunk=dpc, raw_block=block)
    if comp == "LZ4_LENGTH_PREFIXED":           # the writer prefixes the true length: write the wrong one over it
        off0 = int.from_bytes(col.forward_index[28:32].tobytes(), "big")
        col.forward_index[off0:off0 + 4] = np.frombuffer(bad[:4], np.uint8)
    with _group([make_segment("bad", cols + [col])]) as g:
        with pytest.raises(native.PinotB200Error) as e:
            native.execute(g, parse_sql("SELECT blk, SUM(k) FROM t GROUP BY blk LIMIT 100000"), 0)
        assert e.value.code == PB_ERR_INVALID and "do not decode" in str(e.value), str(e.value)
