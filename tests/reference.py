"""An exact, independent restatement of a query over plain value arrays: the reference the device results are held to.

A table is a mapping from column name to `Col` (values, data type, dictionary or raw).  A test that generates its data
hands the reference the values it generated, so the segment writer and the device's decoding are under test too;
`SegmentSource` decodes a segment's columns for tests that only hold the segment.

Per group the reference keeps COUNT; SUM and AVG as (exact sum, n, sum of |x|); MIN and MAX with the group-by semantics
(strict compare, a NaN never enters, defaults +inf / -inf; the device's keyless aggregation does the same, DESIGN §4.5);
DISTINCTCOUNT as the number of distinct values (FLOAT / DOUBLE by the bit pattern of the value widened to double).
`assert_matches_reference` states what a correct device result must satisfy for any summation order.
"""
import dataclasses
import math
import operator as o
from collections.abc import Mapping
from fractions import Fraction
from typing import Dict, NamedTuple, Optional

import numpy as np

from pinot_b200.query import AggOp, And, Not, Or, PredicateType
from pinot_b200.segment_writer import DataType, unpack_bits_be

U = 2.0 ** -53                   # unit roundoff of double, round to nearest


class Col(NamedTuple):
    """values: int64 for INT / LONG, float64 for FLOAT (the float32 values widened) / DOUBLE, bytes ("S") for STRING"""
    values: np.ndarray
    data_type: DataType
    has_dictionary: bool = True


# ---- decoding a segment's columns (the writer's layouts) ----

def _dict_ids(c):
    if c.is_sorted:
        pairs = np.frombuffer(c.forward_index.tobytes(), dtype=">i4").reshape(-1, 2)
        ids = np.zeros(c.num_docs, np.int64)
        for d, (s, e) in enumerate(pairs):
            ids[s:e + 1] = d
        return ids
    return unpack_bits_be(c.forward_index, c.num_docs, c.bits_per_element).astype(np.int64)


def _raw_values(c):
    """the values of a PASS_THROUGH raw column: the last num_docs fixed-width entries of its forward index"""
    dt = {DataType.INT: ">i4", DataType.LONG: ">i8", DataType.FLOAT: ">f4", DataType.DOUBLE: ">f8"}[c.data_type]
    width = np.dtype(dt).itemsize
    return np.frombuffer(c.forward_index.tobytes()[-width * c.num_docs:], dtype=dt)


def raw_is_compressed(c) -> bool:
    """a chunk-compressed raw forward index (header int 5 = compression type)"""
    return not c.has_dictionary and int(np.frombuffer(c.forward_index[20:24].tobytes(), dtype=">i4")[0]) != 0


def _column_values(seg, col):
    c = seg.columns[col]
    if not c.has_dictionary:
        v = _raw_values(c)
        return v.astype(np.float64) if c.data_type in (DataType.FLOAT, DataType.DOUBLE) else v.astype(np.int64)
    d = c.dictionary_values()
    ids = _dict_ids(c)
    if c.data_type == DataType.STRING:
        return np.array(list(d), dtype="S")[ids]                     # bytes: same order as Java compareTo for ASCII
    return d.astype(np.int64)[ids] if c.data_type in (DataType.INT, DataType.LONG) else d.astype(np.float64)[ids]


class SegmentSource(Mapping):
    """A segment's columns as a reference table, decoded on first use"""

    def __init__(self, seg):
        self.seg, self.num_docs, self._cache = seg, seg.num_docs, {}

    def __getitem__(self, name):
        if name not in self._cache:
            c = self.seg.columns[name]
            self._cache[name] = Col(_column_values(self.seg, name), c.data_type, c.has_dictionary)
        return self._cache[name]

    def __iter__(self):
        return iter(self.seg.columns)

    def __len__(self):
        return len(self.seg.columns)


def _table(t):
    return SegmentSource(t) if hasattr(t, "columns") and hasattr(t, "num_docs") else t


def _num_docs(t) -> int:
    return t.num_docs if hasattr(t, "num_docs") else len(next(iter(t.values())).values)


# ---- the WHERE / FILTER tree ----

def evaluate_sql(table, node):
    """The WHERE tree straight from the SQL semantics on the column values (no dictIds, no indexes).  `table`: a mapping
    from column name to Col, or a segment."""
    table = _table(table)
    if node is None:
        return np.ones(_num_docs(table), bool)
    if isinstance(node, (And, Or)):
        parts = [evaluate_sql(table, c) for c in node.children]
        return np.logical_and.reduce(parts) if isinstance(node, And) else np.logical_or.reduce(parts)
    if isinstance(node, Not):
        return ~evaluate_sql(table, node.child)
    c = table[node.column]
    v = c.values

    def lit(s):
        if c.data_type == DataType.STRING:
            return s.encode()
        return float(s) if c.data_type in (DataType.FLOAT, DataType.DOUBLE) else int(s)

    def cmp(op, x):
        return op(v, np.bytes_(x)) if c.data_type == DataType.STRING else op(v, x)
    t = node.type
    if t in (PredicateType.EQ, PredicateType.NOT_EQ):
        m = cmp(o.eq, lit(node.values[0]))
        return ~m if t == PredicateType.NOT_EQ else m
    if t in (PredicateType.IN, PredicateType.NOT_IN):
        if not c.has_dictionary and c.data_type in (DataType.FLOAT, DataType.DOUBLE):
            # a fastutil DoubleSet compares Double.doubleToLongBits (-0.0 is not in {0.0}); EQ / NOT_EQ above compare with ==
            bits = v.astype(np.float64).view(np.int64)
            lits = [np.float32(x) if c.data_type == DataType.FLOAT else np.float64(x) for x in node.values]
            m = np.isin(bits, np.array([np.float64(x) for x in lits]).view(np.int64))
        else:
            m = np.logical_or.reduce([cmp(o.eq, lit(x)) for x in node.values])
        return ~m if t == PredicateType.NOT_IN else m
    m = np.ones(len(v), bool)
    if node.lower is not None:
        m &= cmp(o.ge if node.lower_inclusive else o.gt, lit(node.lower))
    if node.upper is not None:
        m &= cmp(o.le if node.upper_inclusive else o.lt, lit(node.upper))
    return m


# ---- aggregation ----

class SumRef(NamedTuple):
    exact: object                # int for INT / LONG inputs, else math.fsum (correctly rounded); nan / +-inf when non-finite
    n: int
    abs_sum: float
    max_abs: float
    integral: bool


def _codes(c: Col) -> np.ndarray:
    """dense int codes of a column's values (FLOAT / DOUBLE by bit pattern)"""
    v = c.values.astype(np.float64).view(np.int64) if c.data_type in (DataType.FLOAT, DataType.DOUBLE) else c.values
    return np.unique(v, return_inverse=True)[1].reshape(-1)


def _key_of(c: Col, x):
    if c.data_type in (DataType.INT, DataType.LONG):
        return int(x)
    if c.data_type == DataType.STRING:
        return bytes(x)
    return float(x)


def reference(table, q, first_groups: Optional[int] = None) -> Dict[tuple, list]:
    """key -> per aggregation: COUNT int, SUM / AVG SumRef, MIN / MAX float, DISTINCTCOUNT int.  Every group the main
    filter leaves docs in exists (FILTER clauses do not create or remove groups); keyless: the one row () always.
    first_groups: keep only the groups of the first that many distinct keys in doc order among the docs the main filter
    keeps, with their full aggregates (a key generator that creates groups first come first served)."""
    table = _table(table)
    n = _num_docs(table)
    main = evaluate_sql(table, q.filter)
    docs = np.flatnonzero(main)
    keys = [table[k] for k in q.group_by]
    if keys:
        codes = [_codes(k)[docs] for k in keys]
        gid = np.unique(np.stack(codes, 1), axis=0, return_inverse=True)[1].reshape(-1) if docs.size else np.zeros(0, np.int64)
        n_groups = int(gid.max()) + 1 if docs.size else 0
        first = np.full(n_groups, -1, np.int64)
        first[gid[::-1]] = docs[::-1]
        group_keys = [tuple(_key_of(k, k.values[d]) for k in keys) for d in first]
    else:
        gid = np.zeros(docs.size, np.int64)
        n_groups = 1
        group_keys = [()]
    out = {k: [] for k in group_keys}
    for agg in q.aggregations:
        m = main & evaluate_sql(table, agg.filter) if agg.filter is not None else main
        sel = m[docs]
        g = gid[sel]
        cnt = np.bincount(g, minlength=n_groups)
        if agg.op == AggOp.COUNT:
            vals = [int(x) for x in cnt]
        elif agg.op == AggOp.DISTINCTCOUNT:
            c = table[agg.column]
            pair = np.unique(np.stack([g, _codes(c)[docs][sel]], 1), axis=0) if g.size else np.zeros((0, 2), np.int64)
            vals = [int(x) for x in np.bincount(pair[:, 0], minlength=n_groups)]
        else:
            c = table[agg.column]
            x = c.values[docs][sel]
            order = np.argsort(g, kind="stable")
            g_s, x_s = g[order], x[order]
            starts = np.searchsorted(g_s, np.arange(n_groups))
            nz = cnt > 0                          # the groups with inputs tile x_s in order: reduceat over their starts
            idx = starts[nz]

            def per_group(ufunc, arr, empty):
                r = np.full(n_groups, empty, dtype=arr.dtype)
                if idx.size:
                    r[nz] = ufunc.reduceat(arr, idx)
                return r
            if agg.op in (AggOp.MIN, AggOp.MAX):
                fill = np.inf if agg.op == AggOp.MIN else -np.inf
                xf = x_s.astype(np.float64)
                xf = np.where(np.isnan(xf), fill, xf)             # a NaN never enters
                vals = per_group(np.minimum if agg.op == AggOp.MIN else np.maximum, xf, fill).tolist()
            elif c.data_type in (DataType.INT, DataType.LONG):
                xi = x_s.astype(np.int64)
                a = np.abs(xi.astype(np.float64))
                abs_sum, max_abs = per_group(np.add, a, 0.0), per_group(np.maximum, a, 0.0)
                wide = abs_sum.max(initial=0.0) >= 2.0 ** 62         # an int64 sum could wrap: Python ints
                tot = per_group(np.add, xi.astype(object) if wide else xi, 0)
                vals = [SumRef(int(tot[i]), int(cnt[i]), float(abs_sum[i]), float(max_abs[i]), True) for i in range(n_groups)]
            else:
                f = x_s.astype(np.float64)
                fin = np.where(np.isfinite(f), f, 0.0)
                a = np.abs(fin)
                abs_sum, max_abs = per_group(np.add, a, 0.0), per_group(np.maximum, a, 0.0)
                n_nan = per_group(np.add, np.isnan(f).astype(np.int64), 0)
                n_pinf = per_group(np.add, (f == np.inf).astype(np.int64), 0)
                n_ninf = per_group(np.add, (f == -np.inf).astype(np.int64), 0)
                naive = per_group(np.add, fin, 0.0)              # one or two terms: the double sum is correctly rounded
                vals = []
                for i in range(n_groups):
                    if n_nan[i] or (n_pinf[i] and n_ninf[i]):
                        ex = math.nan
                    elif n_pinf[i] or n_ninf[i]:
                        ex = math.inf if n_pinf[i] else -math.inf
                    else:
                        ex = float(naive[i]) if cnt[i] <= 2 else math.fsum(fin[starts[i]:starts[i] + cnt[i]].tolist())
                    vals.append(SumRef(ex, int(cnt[i]), float(abs_sum[i]), float(max_abs[i]), False))
        for k, v in zip(group_keys, vals):
            out[k].append(v)
    if first_groups is not None and keys:
        admitted = np.argsort(first, kind="stable")[:first_groups]
        out = {group_keys[g]: out[group_keys[g]] for g in admitted}
    return out


# ---- numGroupsLimit ----

class LimitRef(NamedTuple):
    rows: Dict[tuple, list]      # exact: the groups the device hands back; else a superset of them
    exact: bool
    at_most: int                 # the device hands back at most this many groups
    reached: Optional[bool]      # the num_groups_limit_reached the device must report (None: either)


def limit_reference(table, q, mode: str, key_space: int = 0) -> LimitRef:
    """What a table under q.num_groups_limit hands back (before any ORDER BY trim), DESIGN.md §4.5.  The flag follows
    GroupByOperator.java:116: the key generator's group count (at most the limit) reached the limit.
    mode 'dense': a dense per-segment table, or a combined call over one segment; key_space = the product of the segment's
      dictionary cardinalities of the key columns.  Below it the key generator creates groups first come first served
      (IntMapBasedHolder, DictionaryBasedGroupKeyGenerator.java:1023-1058): the first `limit` keys in doc order, complete.
    mode 'merged': a dense table over several segments merged on the device: every group (a superset of what Pinot keeps).
    mode 'hash': the limit in thread order -- at most `limit` groups, each complete; when there are at least `limit` groups
      the flag is set.  (A ticket lost to a racing claim may refuse a key below the limit: then the flag is set too, so a
      result without the flag holds every group.)"""
    limit = max(1, q.num_groups_limit)
    full = reference(table, q)
    n = len(full) if q.group_by else 0
    if mode == "dense" and limit < key_space:
        return LimitRef(reference(table, q, first_groups=limit), True, limit, n >= limit)
    if mode == "hash":
        return LimitRef(full, False, limit, True if n >= limit else None)
    return LimitRef(full, True, max(n, 1), n >= limit)


def assert_limit_matches(got_rows: Dict[tuple, list], got_reached: int, lref: LimitRef, q, what=""):
    """the group set and the flag against limit_reference (before any trim), every returned group complete"""
    assert got_reached in (0, 1) and (lref.reached is None or bool(got_reached) == lref.reached), \
        f"{what}: num_groups_limit_reached {got_reached}, expected {int(lref.reached)}"
    assert len(got_rows) <= lref.at_most, f"{what}: {len(got_rows)} groups > {lref.at_most}"
    if lref.exact or not got_reached:
        assert_matches_reference(got_rows, lref.rows, q, what)
    else:
        extra = [k for k in got_rows if k not in lref.rows]
        assert not extra, f"{what}: groups not in the reference: {extra[:3]}"
        assert_matches_reference(got_rows, {k: lref.rows[k] for k in got_rows}, q, what)


# ---- the ORDER BY ... LIMIT trim ----
# TableResizer orders the groups by the first ORDER BY expression: a group-by column by its value, an aggregation by its
# final result (AggregationFunction.extractFinalResult).  Values in one int order (larger = better for DESC):
#   INT / LONG keys and COUNT: the integer; STRING keys: byte order (Java compareTo for ASCII);
#   FLOAT / DOUBLE keys and SUM / AVG / MIN / MAX results: Double.compare (-0.0 < 0.0, NaN above +inf);
#   MIN / MAX of a group without input: the +inf / -inf the hand-back emits (MinAggregationFunction / MaxAggregationFunction
#   defaults); AVG of a group without input: AvgAggregationFunction.DEFAULT_FINAL_RESULT = Double.NEGATIVE_INFINITY.
# Where the device's value is not exact (a float SUM / AVG), the order value is the interval every possible device value
# lies in: check_sum's bound, plus one rounding for AVG's division.

def order_double(x: float) -> int:
    """Double.compare order as a signed int"""
    if math.isnan(x):
        return 0x7ff8000000000000
    b = int(np.float64(x).view(np.int64))
    return b if b >= 0 else b ^ 0x7fffffffffffffff


def order_interval(q, key: tuple, row: list):
    """(lo, hi) of the group's first ORDER BY value (a point where the device's value is exact)"""
    kind, idx, _ = q.order_by[0]
    if kind == 0:
        v = key[idx]
        v = order_double(v) if isinstance(v, float) else v
        return v, v
    agg, r = q.aggregations[idx], row[idx]
    if agg.op == AggOp.COUNT:
        return r, r
    if agg.op in (AggOp.MIN, AggOp.MAX):
        # a zero result is either zero: the strict compare keeps a group's first zero, and doc order is the device's to choose
        return (order_double(-0.0), order_double(0.0)) if r == 0 else (order_double(r), order_double(r))
    avg = agg.op == AggOp.AVG
    ex = r.exact
    if avg and r.n == 0:
        v = order_double(-math.inf)
        return v, v
    if isinstance(ex, float) and not math.isfinite(ex):
        v = order_double(ex)                       # (an infinite or NaN sum over n inputs: the average too)
        return v, v
    if r.integral and r.n * r.max_abs < 2.0 ** 53:  # every partial sum exact: the device's sum is exact, AVG one division
        v = order_double(float(ex) / r.n if avg else float(ex))
        return v, v
    b = sum_bound(r)
    lo, hi = float(ex) - b, float(ex) + b
    if avg:
        lo, hi = lo / r.n, hi / r.n
    return order_double(lo - abs(lo) * 4 * U - 5e-324), order_double(hi + abs(hi) * 4 * U + 5e-324)


def trim_bounds(lo, hi, size: int):
    """(must, never) masks over groups with order intervals [lo, hi] (larger = better), keeping the `size` best with ties:
    a group fewer than `size` others could beat must be kept; a group at least `size` others certainly beat is never kept.
    With points both reduce to {g : v(g) >= v(size-th best)}."""
    lo, hi = np.asarray(lo), np.asarray(hi)
    n = len(lo)
    could = n - np.searchsorted(np.sort(hi), lo, side="right") - (hi > lo)        # others h with hi_h > lo_g
    certain = n - np.searchsorted(np.sort(lo), hi, side="right")                  # others h with lo_h > hi_g
    return could < size, certain >= size


def assert_trim_matches_reference(got_rows: Dict[tuple, list], ref: Dict[tuple, list], q, combined: bool, what="", complete=True):
    """The returned groups are reference groups with matching values, and the trim kept the right ones: all of them when
    no trim applies (at most the threshold or the trim size of groups: q.trim(combined)), else by trim_bounds.
    complete=False: `ref` is a superset of the groups the trim ranked (a hash table that reached numGroupsLimit): the
    returned groups are only checked for membership and values."""
    extra = [k for k in got_rows if k not in ref]
    assert not extra, f"{what}: groups not in the reference: {extra[:3]}"
    assert_matches_reference(got_rows, {k: ref[k] for k in got_rows}, q, what)
    size, thr = q.trim(combined)
    if not complete:
        return
    if not size or len(ref) <= thr or len(ref) <= size:
        assert len(got_rows) == len(ref), f"{what}: no trim applies to {len(ref)} groups, {len(got_rows)} returned"
        return
    keys = list(ref)
    iv = [order_interval(q, k, ref[k]) for k in keys]
    if isinstance(iv[0][0], bytes):                # STRING keys: their rank
        rank = {v: i for i, v in enumerate(sorted({a for a, _ in iv}))}
        iv = [(rank[a], rank[b]) for a, b in iv]
    lo = np.array([a for a, _ in iv], dtype=np.int64)
    hi = np.array([b for _, b in iv], dtype=np.int64)
    if not q.order_by[0][2]:                       # ASC: smaller is better
        lo, hi = ~hi, ~lo
    must, never = trim_bounds(lo, hi, size)
    kept = np.array([k in got_rows for k in keys])
    missing = [keys[i] for i in np.flatnonzero(must & ~kept)]
    wrong = [keys[i] for i in np.flatnonzero(never & kept)]
    assert not missing and not wrong, f"{what}: trim to {size} of {len(ref)} groups kept {kept.sum()}: " \
        f"missing {missing[:3]} (order {[order_interval(q, k, ref[k]) for k in missing[:3]]}), " \
        f"kept beaten {wrong[:3]} (order {[order_interval(q, k, ref[k]) for k in wrong[:3]]})"


def concat(tables, columns=None) -> Dict[str, Col]:
    """the docs of several tables one after the other (the merged table of PB_Q_COMBINE); `columns`: only those"""
    tables = [_table(t) for t in tables]
    names = set(columns) if columns is not None else set(tables[0])
    for t in tables[1:]:
        names &= set(t)
    return {c: Col(np.concatenate([t[c].values for t in tables]), tables[0][c].data_type, tables[0][c].has_dictionary) for c in names}


# ---- comparison ----

def keyless_nan_minmax(q, tables) -> set:
    """the keyless MIN / MAX aggregations over inputs that hold a NaN somewhere in the tables: there the oracle folds with
    Math.min / Math.max (the result is NaN), while the device and this reference keep the group-by semantics (DESIGN §4.5)"""
    if q.group_by:
        return set()
    tables = [_table(t) for t in tables]
    return {a for a, agg in enumerate(q.aggregations)
            if agg.op in (AggOp.MIN, AggOp.MAX) and any(np.isnan(t[agg.column].values.astype(np.float64)).any() for t in tables)}


def without_aggregations(got: Dict[tuple, list], exp: Dict[tuple, list], q, skip):
    """(got, exp, q) with the aggregations in `skip` taken out of the rows and the query"""
    keep = [a for a in range(len(q.aggregations)) if a not in skip]
    q2 = dataclasses.replace(q, aggregations=[q.aggregations[a] for a in keep])
    return {k: [r[a] for a in keep] for k, r in got.items()}, {k: [r[a] for a in keep] for k, r in exp.items()}, q2


def sum_bound(r: SumRef) -> float:
    """largest |got - exact| any summation order can produce: gamma_(n-1) * sum|x| + u * |exact|"""
    k = max(r.n - 1, 0) * U
    return k / (1.0 - k) * r.abs_sum + U * abs(float(r.exact))


def check_sum(got: float, r: SumRef) -> Optional[str]:
    """None when `got` is a possible double sum of the inputs, else why not"""
    ex = r.exact
    if isinstance(ex, float) and math.isnan(ex):
        return None if math.isnan(got) else f"{got!r} should be NaN"
    if isinstance(ex, float) and math.isinf(ex):
        return None if got == ex else f"{got!r} should be {ex!r}"
    if math.isnan(got) or math.isinf(got):
        return f"{got!r} from finite inputs (exact {ex!r})"
    if r.integral and r.n * r.max_abs < 2.0 ** 53:
        return None if got == ex else f"{got!r} != {ex} exactly (integers, n*max|x| < 2^53)"
    err = float(abs(Fraction(got) - Fraction(ex)))
    return None if err <= sum_bound(r) else f"{got!r} off by {err:.3g} > bound {sum_bound(r):.3g} (exact {ex!r}, n={r.n})"


def _same_bits(a: float, b: float) -> bool:
    return a == b == 0.0 or np.float64(a).view(np.int64) == np.float64(b).view(np.int64)


def assert_matches_reference(got_rows: Dict[tuple, list], ref: Dict[tuple, list], q, what=""):
    """COUNT, DISTINCTCOUNT and the AVG count exactly; SUM / AVG within the bound of check_sum; MIN / MAX bit for bit
    (+0.0 == -0.0: with a strict compare the first zero of a group wins, and doc order is the device's to choose)"""
    assert set(got_rows) == set(ref), f"{what}: group sets differ: {len(got_rows)} vs {len(ref)}; " \
        f"missing={list(set(ref) - set(got_rows))[:3]} extra={list(set(got_rows) - set(ref))[:3]}"
    for k, erow in ref.items():
        grow = got_rows[k]
        for a, agg in enumerate(q.aggregations):
            g, e = grow[a], erow[a]
            if agg.op in (AggOp.COUNT, AggOp.DISTINCTCOUNT):
                assert g == e, f"{what}: {k} {agg}: {g} != {e}"
            elif agg.op in (AggOp.MIN, AggOp.MAX):
                assert _same_bits(g, e), f"{what}: {k} {agg}: {g!r} != {e!r}"
            else:
                s = g[0] if agg.op == AggOp.AVG else g
                if agg.op == AggOp.AVG:
                    assert g[1] == e.n, f"{what}: {k} {agg}: count {g[1]} != {e.n}"
                why = check_sum(s, e)
                assert why is None, f"{what}: {k} {agg}: {why}"
