"""Seeded generators of fuzz tables and queries for the device differential fuzz (tests/test_gpu_fuzz.py) and for the CPU check
of the reference against the oracle (tests/test_cpu_reference.py).  Deterministic, no network.

A table is a list of segments plus, per segment, the source values the segment was written from (tests/reference.Col), so
the reference never reads a value back from a segment.  The columns and distributions aim at the places where the device's
kernel choices have edges: row groups of 4 and 8 bytes per value, exact-integer sums on both sides of their condition, dense
tables at and past 2^24 slots, 64 / 65-bit hash keys, raw keys, more than 16 segments,
segment sizes at the ends of 1024-doc chunks and 2-chunk units, and IEEE edge values in MIN / MAX inputs.
"""
from typing import Dict, List, Tuple

import numpy as np

from pinot_b200.segment_writer import DataType, build_column, build_dict_column, make_segment
from tests.reference import Col

EDGE_SIZES = (1, 31, 32, 33, 1023, 1024, 1025, 2047, 2049, 4097)
I32 = 2 ** 31
# a DOUBLE dictionary in Double.compare order: both zeros, both infinities, NaN, subnormals and the extremes.  A value-based
# np.unique would fold the zeros into one entry, so the dictionary is written as is (build_dict_column).
EDGE_DOUBLES = np.array([-np.inf, -np.finfo(np.float64).max, -1.5, -5e-324, -0.0, 0.0, 5e-324, 2.2250738585072014e-308, 2.5,
                         np.finfo(np.float64).max, np.inf, np.nan])
NEG_DOUBLES = np.array([-1e300, -7.25, -1.0, -2.5e-300, -5e-324])       # all-negative MAX groups: the result is negative
WIDE = 4096                      # key cardinality: 4096 x 4096 = 2^24 slots, 4096 x 4097 one more (hash)


def _dict_col(name, dt, dict_values, ids, inverted=False, var_length=False):
    """A dictionary column from an explicit sorted dictionary.  When the ids happen to be non-decreasing the writer stores a
    sorted column, which needs every entry to occur: shrink the dictionary to the entries used."""
    ids = np.asarray(ids, dtype=np.int64)
    if ids.size <= 1 or (ids[1:] >= ids[:-1]).all():
        used, ids = np.unique(ids, return_inverse=True)
        dict_values = dict_values[used]
    return build_dict_column(name, dt, dict_values, ids.astype(np.uint32), inverted=inverted, var_length_dictionary=var_length)


def _src(dt, dict_values, ids):
    v = dict_values[np.asarray(ids, dtype=np.int64)]
    if dt == DataType.STRING:
        return Col(np.array(list(v), dtype="S"), dt, True)
    return Col(v.astype(np.int64) if dt in (DataType.INT, DataType.LONG) else v.astype(np.float64), dt, True)


def segment_sizes(rng, seed: int, max_total: int) -> List[int]:
    # every fourth seed puts more than 16 segments in one call (pb_agg_rows_kernel then reads its descriptors from global memory)
    n_segs = int(rng.choice([17, 20, 24])) if seed % 4 == 1 else int(rng.choice([1, 2, 3, 5, 8]))
    sizes = []
    for _ in range(n_segs):
        sizes.append(int(rng.choice(EDGE_SIZES)) if rng.random() < 0.6 else int(rng.integers(5_000, 300_000)))
    while sum(sizes) > max_total:
        i = int(np.argmax(sizes))
        sizes[i] = max(1, sizes[i] // 3)
    return sizes


def make_tables(seed: int, max_total: int = 600_000, sizes: List[int] = None) -> Tuple[list, List[Dict[str, Col]], dict]:
    """(segments, per-segment source columns, facts about the table the tests use); sizes: the docs of each segment, in
    place of the seed's choice"""
    rng = np.random.default_rng(77_000 + seed)
    sizes = segment_sizes(rng, seed, max_total) if sizes is None else list(sizes)
    total = sum(sizes)
    # LONG metric: max|v| x docs of the whole call just inside or just outside 2^53 (plan_rows_kernel's exact-integer test)
    long_bound = int((2 ** 53) // total * (0.5 if seed % 2 == 0 else 2.0))
    long_dict = np.unique(np.concatenate([rng.integers(-long_bound, long_bound, 200), [-long_bound, long_bound]])).astype(np.int64)
    int_dict = np.unique(np.concatenate([rng.integers(-I32, -I32 + 1000, 40), rng.integers(I32 - 1000, I32, 40),
                                         rng.integers(-1000, 1000, 40)])).astype(np.int64)
    mixed_dict = np.unique(np.concatenate([rng.integers(-3, 4, 20) * 1e15, rng.normal(0, 1, 60)]))   # 1e15 and 1: cancellation
    flt_dict = np.unique(rng.normal(0, 100, 300).astype(np.float32))
    str_dict = np.array(sorted({f"s{int(x):03d}".encode() for x in rng.integers(0, 60, 80)}), dtype=object)
    wide_card = WIDE + (1 if seed % 3 == 2 else 0)
    budget_card = 17_066 + (seed % 2)          # ~17 k slots: a CTA table only for narrow queries (the budget edge itself:
                                               # test_gpu_fuzz.py::test_cta_table_at_the_shared_memory_budget)
    sorted_card = 50
    segs, srcs = [], []
    for si, n in enumerate(sizes):
        r = np.random.default_rng([seed, si])
        cols, src = [], {}

        def add(name, dt, dvals, ids, **kw):
            cols.append(_dict_col(name, dt, dvals, ids, **kw))
            src[name] = _src(dt, dvals, ids)

        def add_raw(name, dt, values, compression=None):
            cols.append(build_column(name, dt, values, dictionary=False, raw_compression=compression))
            src[name] = Col(np.asarray(values).astype(np.float64 if dt in (DataType.FLOAT, DataType.DOUBLE) else np.int64), dt, False)
        # keys
        add("k3", DataType.INT, np.array([-5, 0, 7], dtype=np.int64), r.integers(0, 3, n))
        add("k2", DataType.INT, np.array([10, 20], dtype=np.int64), r.integers(0, 2, n))
        add("kstr", DataType.STRING, str_dict, r.integers(0, len(str_dict), n), var_length=(seed % 2 == 1))
        add("kwa", DataType.INT, np.arange(WIDE, dtype=np.int64) * 3, r.integers(0, WIDE, n))
        add("kwb", DataType.LONG, np.arange(wide_card, dtype=np.int64) - 2000, r.integers(0, wide_card, n))
        add("kbud", DataType.INT, np.arange(budget_card, dtype=np.int64), r.integers(0, budget_card, n))
        add_raw("rki", DataType.INT, r.integers(-50, 50, n).astype(np.int32))
        add_raw("rkj", DataType.INT, r.integers(-3, 3, n).astype(np.int32))
        add_raw("rkl", DataType.LONG, r.integers(-2, 2, n).astype(np.int64) * (2 ** 40))
        # filter columns
        sv = np.sort(r.integers(0, sorted_card, n))
        cols.append(build_column("fsort", DataType.INT, sv.astype(np.int32)))
        src["fsort"] = Col(sv.astype(np.int64), DataType.INT, True)
        add("finv", DataType.INT, np.arange(200, dtype=np.int64), r.integers(0, 200, n), inverted=True)
        add("fu", DataType.INT, np.arange(1000, dtype=np.int64) * 2, r.integers(0, 1000, n))
        # metrics
        add("mint", DataType.INT, int_dict, r.integers(0, len(int_dict), n))
        add("mlong", DataType.LONG, long_dict, r.integers(0, len(long_dict), n))
        add("mdbl", DataType.DOUBLE, mixed_dict, r.integers(0, len(mixed_dict), n))
        add("mflt", DataType.FLOAT, flt_dict, r.integers(0, len(flt_dict), n))
        add("edbl", DataType.DOUBLE, EDGE_DOUBLES, r.integers(0, len(EDGE_DOUBLES), n))       # MIN / MAX only
        add("eneg", DataType.DOUBLE, NEG_DOUBLES, r.integers(0, len(NEG_DOUBLES), n))
        add("enan", DataType.DOUBLE, np.array([np.nan]), np.zeros(n, np.int64))               # every input NaN
        add_raw("rint", DataType.INT, r.integers(-I32, I32, n).astype(np.int32))
        add_raw("rlong", DataType.LONG, r.integers(-(2 ** 40), 2 ** 40, n))
        add_raw("rflt", DataType.FLOAT, r.normal(0, 10, n).astype(np.float32))
        add_raw("rdbl", DataType.DOUBLE, np.round(r.normal(0, 1e6, n), 3))
        add_raw("redge", DataType.DOUBLE, EDGE_DOUBLES[r.integers(0, len(EDGE_DOUBLES), n)])    # MIN / MAX only
        add_raw("rz", DataType.DOUBLE, np.round(r.normal(0, 50, n), 2), compression="LZ4" if seed % 2 else "SNAPPY")
        segs.append(make_segment(f"fz{seed}_{si}", cols))
        srcs.append(src)
    return segs, srcs, {"sizes": sizes, "wide_card": wide_card, "budget_card": budget_card, "long_bound": long_bound}


SUM_COLS = ["mint", "mlong", "mdbl", "mflt", "rint", "rlong", "rflt", "rdbl", "rz", "fu"]
MINMAX_COLS = SUM_COLS + ["edbl", "eneg", "enan", "redge"]
DC_COLS = ["mint", "mlong", "kstr", "fu", "rint", "rdbl", "mflt"]
# (at most ~100 bits of scanned columns per row fit the filter kernel's unit stages: wider trees are declined)
FILTER_COLS = ["fsort", "finv", "fu", "k3", "kstr", "mint", "rint", "mflt"]
# group-by shapes, each a planner edge (comments: what the planner picks)
KEY_SETS = [
    [],                                   # keyless
    ["k3"], ["k2", "k3"],                 # small dense tables: many CTA-table replicas
    ["kstr"], ["k3", "kstr"],
    ["kbud"],                             # ~17 k dense slots: mostly past the shared-memory budget (global table)
    ["kwa", "kwb"],                       # 4096 x 4096 = 2^24 slots (dense) or 4096 x 4097 (hash, 25 bits)
    ["rki", "rkj"],                       # raw keys: 64 bits, one key word
    ["rki", "rkj", "k2"],                 # 65 bits: two key words
    ["rkl", "rki", "k3", "kstr"], ["rkl"], ["k3", "k2", "kstr", "finv", "fsort"],
]


def _literal(rng, src: Col) -> str:
    v = src.values[int(rng.integers(0, len(src.values)))]
    if src.data_type == DataType.STRING:
        return "'" + bytes(v).decode() + "'"
    if src.data_type in (DataType.FLOAT, DataType.DOUBLE):
        return repr(float(v))
    return str(int(v) + int(rng.choice([0, 0, 1, -1])))


def _predicate(rng, src: Dict[str, Col], col: str) -> str:
    kind = rng.choice(["eq", "neq", "in", "notin", "lt", "ge", "between"])
    lit = lambda: _literal(rng, src[col])
    if kind == "eq":
        return f"{col} = {lit()}"
    if kind == "neq":
        return f"{col} <> {lit()}"
    if kind in ("in", "notin"):
        return f"{col} {'NOT IN' if kind == 'notin' else 'IN'} ({', '.join(lit() for _ in range(int(rng.integers(1, 6))))})"
    if kind == "between":
        a, b = sorted([lit(), lit()], key=lambda s: float(s.strip("'")) if "'" not in s else 0)
        return f"{col} BETWEEN {a} AND {b}"
    return f"{col} {'<' if kind == 'lt' else '>='} {lit()}"


def _expr(rng, src, depth):
    if depth == 0 or rng.random() < 0.35:
        return _predicate(rng, src, str(rng.choice(FILTER_COLS)))
    op = " AND " if rng.random() < 0.5 else " OR "
    return "(" + op.join(_expr(rng, src, depth - 1) for _ in range(int(rng.integers(2, 4)))) + ")"


def where_clause(rng, src: Dict[str, Col]) -> str:
    """steered: a single dictionary leaf (the specialised filter kernel), a flat conjunction whose best leaf keeps <= 3 %
    of the docs (candidate leaves), match-all, empty, or a random tree"""
    r = rng.random()
    if r < 0.25:
        col = str(rng.choice(["fu", "finv", "k3", "mint"]))
        return f" WHERE {col} IN ({', '.join(_literal(rng, src[col]) for _ in range(int(rng.integers(1, 12))))})" if rng.random() < 0.5 \
            else f" WHERE {col} < {_literal(rng, src[col])}"
    if r < 0.45:
        lo = int(rng.integers(0, 1960))
        return f" WHERE fu BETWEEN {lo} AND {lo + int(rng.integers(0, 40))} AND {_predicate(rng, src, str(rng.choice(['k3', 'mint', 'finv', 'rint'])))}"
    if r < 0.55:
        return ""
    if r < 0.6:
        return " WHERE fu < -5"                        # empty
    return " WHERE " + _expr(rng, src, 2)


def make_query(rng, src: Dict[str, Col]) -> str:
    keys = KEY_SETS[int(rng.integers(0, len(KEY_SETS)))]
    wide = "kwa" in keys or "kbud" in keys          # (a DISTINCTCOUNT bitset per slot of a 2^24-slot table is gigabytes)
    aggs = []
    for _ in range(int(rng.integers(1, 7))):
        op = str(rng.choice(["COUNT", "SUM", "MIN", "MAX", "AVG"] + ([] if wide else ["DISTINCTCOUNT"])))
        col = "*" if op == "COUNT" else str(rng.choice(DC_COLS if op == "DISTINCTCOUNT" else MINMAX_COLS if op in ("MIN", "MAX") else SUM_COLS))
        flt = f" FILTER(WHERE {_expr(rng, src, 1)})" if rng.random() < 0.15 else ""
        aggs.append(f"{op}({col}){flt}")
    gb = f" GROUP BY {', '.join(keys)} LIMIT 100000000" if keys else ""
    return f"SET numGroupsLimit = 100000000; SELECT {', '.join(aggs)} FROM t{where_clause(rng, src)}{gb}"


def make_shaped_query(rng, src: Dict[str, Col]) -> str:
    """A group-by query whose result is shaped on the device: ORDER BY a key column or a (possibly filtered) non-DISTINCTCOUNT
    aggregation, ASC or DESC, LIMIT 1-4 and trim sizes small enough that the trim fires on tables above ~10 groups (and
    stays off on k3 and k2, k3); for about half the queries a numGroupsLimit below the key space.  Its own rng stream
    (make_query's seeds and coverage stay as they are)."""
    keys = KEY_SETS[int(rng.integers(1, len(KEY_SETS)))]
    aggs = []
    for _ in range(int(rng.integers(1, 5))):
        op = str(rng.choice(["COUNT", "SUM", "MIN", "MAX", "AVG"]))
        col = "*" if op == "COUNT" else str(rng.choice(MINMAX_COLS if op in ("MIN", "MAX") else SUM_COLS))
        flt = f" FILTER(WHERE {_expr(rng, src, 1)})" if rng.random() < 0.3 else ""
        aggs.append(f"{op}({col}){flt}")
    if rng.random() < 0.4:
        ob = str(rng.choice(keys))
    else:
        ob = aggs[int(rng.integers(0, len(aggs)))]
    limit = int(rng.integers(1, 5))
    size = int(rng.integers(6, 11))             # (5 x LIMIT is at most 20)
    opts = f"SET minServerGroupTrimSize = {size}; SET minSegmentGroupTrimSize = {size}; " \
           f"SET groupTrimThreshold = {int(rng.integers(1, 3)) * max(size, 5 * limit)}; "
    ngl = int(rng.choice([1, 2, 5, 20, 300])) if rng.random() < 0.5 else 100000000
    return f"SET numGroupsLimit = {ngl}; {opts}SELECT {', '.join(aggs)} FROM t{where_clause(rng, src)} GROUP BY {', '.join(keys)} " \
           f"ORDER BY {ob} {'DESC' if rng.random() < 0.5 else 'ASC'} LIMIT {limit}"


HASH_KEY_SETS = [["rki", "rkj"], ["rkl"],                     # raw keys, one key word
                 ["rki", "rkj", "k2"], ["rkl", "rki", "k3", "kstr"]]     # two key words


def make_hash_query(rng, src: Dict[str, Col], wide_card: int = WIDE) -> str:
    """A query whose group table is a hash table (the hash key sets of KEY_SETS; kwa, kwb when kwb has 4097 values): COUNT /
    SUM / MIN / MAX / AVG, about 30 % of them under a FILTER clause.  Its own rng stream (make_query's seeds and coverage stay
    as they are)."""
    key_sets = HASH_KEY_SETS + ([["kwa", "kwb"]] if wide_card > WIDE else [])
    keys = key_sets[int(rng.integers(0, len(key_sets)))]
    aggs = []
    for _ in range(int(rng.integers(1, 6))):
        op = str(rng.choice(["COUNT", "SUM", "MIN", "MAX", "AVG"]))
        col = "*" if op == "COUNT" else str(rng.choice(MINMAX_COLS if op in ("MIN", "MAX") else SUM_COLS))
        flt = f" FILTER(WHERE {_expr(rng, src, 1)})" if rng.random() < 0.3 else ""
        aggs.append(f"{op}({col}){flt}")
    return f"SET numGroupsLimit = 100000000; SELECT {', '.join(aggs)} FROM t{where_clause(rng, src)} GROUP BY {', '.join(keys)} LIMIT 100000000"
