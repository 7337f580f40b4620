"""ctypes wrapper over oracle/liboracle.so (pinot_oracle.c).

TEST INFRASTRUCTURE ONLY — imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never by the product package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Dict, List, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle.so")
_SRC = [os.path.join(_HERE, "pinot_oracle.c"), os.path.join(_HERE, "pinot_oracle.h")]


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRC if os.path.exists(s)):
        subprocess.check_call(["gcc", "-O3", "-march=native", "-std=gnu11", "-shared", "-fPIC", "-pthread", "-o", _SO, _SRC[0], "-lm"])
    return _SO


class OrcColumn(C.Structure):
    _fields_ = [("data_type", C.c_int32), ("has_dictionary", C.c_int32), ("is_sorted", C.c_int32),
                ("cardinality", C.c_int32), ("bits_per_element", C.c_int32), ("dict_entry_bytes", C.c_int32),
                ("forward_index", C.c_void_p), ("forward_index_len", C.c_int64),
                ("dictionary", C.c_void_p), ("dictionary_len", C.c_int64),
                ("inverted_index", C.c_void_p), ("inverted_index_len", C.c_int64),
                ("null_value_vector", C.c_void_p), ("null_value_vector_len", C.c_int64)]


class OrcSegment(C.Structure):
    _fields_ = [("num_docs", C.c_int32), ("num_columns", C.c_int32), ("columns", C.POINTER(OrcColumn))]


class OrcPredicate(C.Structure):
    _fields_ = [("type", C.c_int32), ("column", C.c_int32), ("num_values", C.c_int32),
                ("lower_unbounded", C.c_int32), ("upper_unbounded", C.c_int32),
                ("lower_inclusive", C.c_int32), ("upper_inclusive", C.c_int32), ("_pad", C.c_int32),
                ("int_values", C.POINTER(C.c_int64)), ("double_values", C.POINTER(C.c_double)),
                ("string_values", C.POINTER(C.c_char_p))]


class OrcFilterNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_children", C.c_int32), ("predicate", C.c_int32)]


class OrcAggregation(C.Structure):
    _fields_ = [("op", C.c_int32), ("column", C.c_int32)]


class OrcFilterProgram(C.Structure):
    _fields_ = [("num_nodes", C.c_int32), ("_pad", C.c_int32),
                ("nodes", C.POINTER(OrcFilterNode)), ("predicates", C.POINTER(OrcPredicate))]


class OrcQuery(C.Structure):
    _fields_ = [("num_filter_nodes", C.c_int32), ("num_group_by", C.c_int32), ("num_aggregations", C.c_int32),
                ("num_groups_limit", C.c_int32), ("max_initial_result_holder_capacity", C.c_int32),
                ("skip_inverted_index", C.c_int32),
                ("filter_nodes", C.POINTER(OrcFilterNode)), ("predicates", C.POINTER(OrcPredicate)),
                ("group_by_columns", C.POINTER(C.c_int32)), ("aggregations", C.POINTER(OrcAggregation)),
                ("num_agg_filters", C.c_int32), ("null_handling", C.c_int32),
                ("agg_filters", C.POINTER(OrcFilterProgram)), ("agg_filter_of", C.POINTER(C.c_int32))]


class OrcStats(C.Structure):
    _fields_ = [("num_docs_scanned", C.c_int64), ("num_entries_scanned_in_filter", C.c_int64),
                ("num_entries_scanned_post_filter", C.c_int64), ("num_total_docs", C.c_int64),
                ("num_groups_limit_reached", C.c_int32), ("key_holder", C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(build())
        l.orc_execute.argtypes = [C.POINTER(OrcSegment), C.POINTER(OrcQuery)]
        l.orc_execute.restype = C.c_void_p
        l.orc_result_free.argtypes = [C.c_void_p]
        l.orc_last_error.restype = C.c_char_p
        l.orc_result_num_groups.argtypes = [C.c_void_p]
        l.orc_result_num_groups.restype = C.c_int32
        l.orc_result_stats.argtypes = [C.c_void_p]
        l.orc_result_stats.restype = C.POINTER(OrcStats)
        l.orc_result_group_keys.argtypes = [C.c_void_p]
        l.orc_result_group_keys.restype = C.POINTER(C.c_int64)
        for fn, rt in (("orc_result_double", C.c_double), ("orc_result_long", C.c_int64),
                       ("orc_result_distinct_offsets", C.c_int64), ("orc_result_distinct_dict_ids", C.c_int32)):
            getattr(l, fn).argtypes = [C.c_void_p, C.c_int32]
            getattr(l, fn).restype = C.POINTER(rt)
        l.orc_filter_doc_ids.argtypes = [C.POINTER(OrcSegment), C.POINTER(OrcQuery), C.POINTER(C.POINTER(C.c_int32)),
                                         C.POINTER(C.c_int64)]
        l.orc_filter_doc_ids.restype = C.c_int64
        l.orc_free.argtypes = [C.c_void_p]
        l.orc_result_distinct_values.argtypes = [C.c_void_p, C.c_int32]
        l.orc_result_distinct_values.restype = C.POINTER(C.c_int64)
        l.orc_execute_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        l.orc_execute_batch.restype = C.c_int32
        l.orc_execute_combined.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        l.orc_execute_combined.restype = C.c_int64
        l.orc_free.argtypes = [C.c_void_p]
        l.orc_num_bits_per_value.argtypes = [C.c_int32]
        l.orc_num_bits_per_value.restype = C.c_int32
        l.orc_read_dict_id.argtypes = [C.c_void_p, C.c_int32, C.c_int64]
        l.orc_read_dict_id.restype = C.c_int32
        l.orc_roaring_to_doc_ids.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        l.orc_roaring_to_doc_ids.restype = C.c_int64
        for f in (l.orc_lz4_block_decode, l.orc_snappy_block_decode):
            f.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
            f.restype = C.c_int64
        l.orc_raw_forward_decompress.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64]
        l.orc_raw_forward_decompress.restype = C.c_int64
        _lib = l
    return _lib


def raw_forward_decompress(fwd: np.ndarray, width: int, num_docs: int = -1) -> np.ndarray:
    """A chunk-compressed raw forward index rewritten as the equivalent PASS_THROUGH one (orc_raw_forward_decompress).
    num_docs: the segment's doc count, which a version 1 index does not hold."""
    fwd = np.ascontiguousarray(fwd, dtype=np.uint8)
    need = lib().orc_raw_forward_decompress(fwd.ctypes.data, fwd.size, width, num_docs, None, 0)
    if need < 0:
        raise RuntimeError(lib().orc_last_error().decode())
    out = np.zeros(need, dtype=np.uint8)
    if lib().orc_raw_forward_decompress(fwd.ctypes.data, fwd.size, width, num_docs, out.ctypes.data, out.size) != need:
        raise RuntimeError(lib().orc_last_error().decode())
    return out


def block_decode(codec: str, data: bytes, decoded_size: int) -> bytes:
    """One LZ4 block / raw Snappy block through the oracle's decoder (tests pin it against pyarrow's codecs)."""
    src = np.frombuffer(data, dtype=np.uint8)
    out = np.zeros(max(decoded_size, 1), dtype=np.uint8)
    f = lib().orc_lz4_block_decode if codec == "lz4" else lib().orc_snappy_block_decode
    n = f(src.ctypes.data, src.size, out.ctypes.data, decoded_size)
    if n < 0:
        raise ValueError("malformed %s block" % codec)
    return out[:n].tobytes()


class _Marshalled:
    """Keeps every ctypes object a call needs alive."""

    def __init__(self):
        self.keep = []

    def hold(self, x):
        self.keep.append(x)
        return x


def marshal_segment(seg, m: _Marshalled, skip_inverted=()) -> OrcSegment:
    cols = (OrcColumn * len(seg.columns))()
    for i, c in enumerate(seg.columns.values()):
        oc = cols[i]
        oc.data_type = int(c.data_type)
        oc.has_dictionary = int(c.has_dictionary)
        oc.is_sorted = int(c.is_sorted and c.has_dictionary)
        oc.cardinality = c.cardinality
        oc.bits_per_element = c.bits_per_element
        oc.dict_entry_bytes = c.dict_entry_bytes
        fwd = c.forward_index
        version = int.from_bytes(fwd[0:4].tobytes(), "big") if not c.has_dictionary else 0
        if not c.has_dictionary and (version == 1 or fwd.size >= 28 and version > 1 and int.from_bytes(fwd[20:24].tobytes(), "big") != 0):
            fwd = m.hold(raw_forward_decompress(fwd, c.dict_entry_bytes, seg.num_docs))   # chunk codec -> plain values (v1: SNAPPY)
        oc.forward_index = fwd.ctypes.data
        oc.forward_index_len = fwd.size
        if c.dictionary is not None:
            oc.dictionary = c.dictionary.ctypes.data
            oc.dictionary_len = c.dictionary.size
        if c.inverted_index is not None and c.name not in skip_inverted:
            oc.inverted_index = c.inverted_index.ctypes.data
            oc.inverted_index_len = c.inverted_index.size
        if getattr(c, "null_value_vector", None) is not None:
            oc.null_value_vector = c.null_value_vector.ctypes.data
            oc.null_value_vector_len = c.null_value_vector.size
    m.hold(cols)
    s = OrcSegment(seg.num_docs, len(seg.columns), cols)
    return m.hold(s)


def _marshal_filter(seg, flt, m: _Marshalled):
    """postfix nodes + predicates of one filter expression -> (n_nodes, OrcFilterNode[], OrcPredicate[])"""
    from pinot_b200.query import postfix_of
    from pinot_b200.segment_writer import DataType
    names = seg.column_names()
    nodes, preds = postfix_of(flt)
    cn = (OrcFilterNode * max(1, len(nodes)))()
    for i, (k, n, p) in enumerate(nodes):
        cn[i].kind, cn[i].n_children, cn[i].predicate = k, n, p
    cp = (OrcPredicate * max(1, len(preds)))()
    for i, p in enumerate(preds):
        col = seg.columns[p.column]
        o = cp[i]
        o.type = int(p.type)
        o.column = names.index(p.column)
        if int(p.type) == 4:
            vals = [p.lower if p.lower is not None else "0", p.upper if p.upper is not None else "0"]
            o.lower_unbounded = int(p.lower is None)
            o.upper_unbounded = int(p.upper is None)
            o.lower_inclusive = int(p.lower_inclusive)
            o.upper_inclusive = int(p.upper_inclusive)
        else:
            vals = list(p.values)
        o.num_values = len(vals)
        if col.data_type in (DataType.INT, DataType.LONG):
            ints = [int(float(v)) if ("." in v or "e" in v.lower()) else int(v) for v in vals]
            if any(not -2**63 <= x < 2**63 for x in ints):      # Long.parseLong would throw: the query fails in the reference
                raise ValueError(f"integral literal out of range in a predicate on {p.column}")
            arr = (C.c_int64 * max(1, len(vals)))(*ints)
            o.int_values = m.hold(arr)
        elif col.data_type in (DataType.FLOAT, DataType.DOUBLE):
            arr = (C.c_double * max(1, len(vals)))(*[float(v) for v in vals])
            o.double_values = m.hold(arr)
        else:
            arr = (C.c_char_p * max(1, len(vals)))(*[v.encode("utf-8") for v in vals])
            o.string_values = m.hold(arr)
    m.hold((cn, cp))
    return len(nodes), cn, cp


def marshal_query(seg, q, m: _Marshalled) -> OrcQuery:
    names = seg.column_names()
    n_nodes, cn, cp = _marshal_filter(seg, q.filter, m)
    nodes = [None] * n_nodes
    gb = (C.c_int32 * max(1, len(q.group_by)))(*[names.index(c) for c in q.group_by])
    ag = (OrcAggregation * max(1, len(q.aggregations)))()
    for i, a in enumerate(q.aggregations):
        ag[i].op = int(a.op)
        keep_col = a.column is not None and (int(a.op) != 0 or getattr(q, "null_handling", False))   # COUNT(col) = COUNT(*) unless nulls are handled
        ag[i].column = names.index(a.column) if keep_col else -1
    filters, filter_of = q.agg_filters()
    progs = (OrcFilterProgram * max(1, len(filters)))()
    for i, f in enumerate(filters):
        n, fn_, fp_ = _marshal_filter(seg, f, m)
        progs[i].num_nodes, progs[i].nodes, progs[i].predicates = n, fn_, fp_
    fo = (C.c_int32 * max(1, len(filter_of)))(*filter_of)
    oq = OrcQuery(len(nodes), len(q.group_by), len(q.aggregations), q.num_groups_limit,
                  q.max_initial_result_holder_capacity, int(q.skip_inverted_all), cn, cp, gb, ag,
                  len(filters), int(getattr(q, "null_handling", False)), progs, fo)
    m.hold((cn, cp, gb, ag, progs, fo))
    return m.hold(oq)


class OracleResult:
    """Per-segment result, copied out of the C result into numpy."""

    def __init__(self, seg, q, rp):
        l = lib()
        self.num_groups = l.orc_result_num_groups(rp)
        st = l.orc_result_stats(rp).contents
        self.stats = {k: getattr(st, k) for k, _ in OrcStats._fields_}
        ng, nG = self.num_groups, len(q.group_by)
        self.group_keys = (np.ctypeslib.as_array(l.orc_result_group_keys(rp), shape=(max(ng, 1) * max(nG, 1),))
                           [:ng * nG].reshape(ng, nG).copy() if nG else np.zeros((ng, 0), dtype=np.int64))
        self.doubles, self.longs, self.distinct = [], [], []
        for a, agg in enumerate(q.aggregations):
            self.doubles.append(np.ctypeslib.as_array(l.orc_result_double(rp, a), shape=(max(ng, 1),))[:ng].copy())
            self.longs.append(np.ctypeslib.as_array(l.orc_result_long(rp, a), shape=(max(ng, 1),))[:ng].copy())
            if int(agg.op) == 5:
                off = np.ctypeslib.as_array(l.orc_result_distinct_offsets(rp, a), shape=(ng + 1,)).copy()
                n = int(off[-1])
                if seg.columns[agg.column].has_dictionary:      # value sets as dictIds ...
                    ids = np.ctypeslib.as_array(l.orc_result_distinct_dict_ids(rp, a), shape=(max(n, 1),))[:n].copy()
                else:                                           # ... or, for a raw column, as value bits (int64)
                    ids = np.ctypeslib.as_array(l.orc_result_distinct_values(rp, a), shape=(max(n, 1),))[:n].copy()
                self.distinct.append((off, ids))
            else:
                self.distinct.append(None)
        self.segment = seg
        self.query = q

    def decoded_keys(self) -> List[tuple]:
        """Group keys decoded to values (GroupKeyGenerator.GroupKey._keys)."""
        out = []
        cols = [self.segment.columns[c] for c in self.query.group_by]
        dicts = [c.dictionary_values() if c.has_dictionary else None for c in cols]
        from pinot_b200.segment_writer import DataType
        for g in range(self.num_groups):
            key = []
            for j, c in enumerate(cols):
                k = int(self.group_keys[g, j])
                if c.has_dictionary:
                    v = dicts[j][k]
                    key.append(v.item() if hasattr(v, "item") else v)
                elif c.data_type in (DataType.FLOAT, DataType.DOUBLE):
                    key.append(float(np.int64(k).view(np.float64)))
                else:
                    key.append(k)
            out.append(tuple(key))
        return out


def execute(seg, q) -> OracleResult:
    """GroupByOperator / AggregationOperator over one segment."""
    m = _Marshalled()
    skip = [c for c, kinds in q.skip_indexes.items() if "inverted" in kinds]
    s = marshal_segment(seg, m, skip_inverted=skip)
    oq = marshal_query(seg, q, m)
    rp = lib().orc_execute(C.byref(s), C.byref(oq))
    if not rp:
        raise RuntimeError("oracle: " + lib().orc_last_error().decode())
    try:
        return OracleResult(seg, q, rp)
    finally:
        lib().orc_result_free(rp)


class PreparedBatch:
    """segments + query marshalled once (what a server does at plan time), for execute_batch"""

    def __init__(self, segs, q):
        self.segs, self.q, self.m = list(segs), q, _Marshalled()
        skip = [c for c, kinds in q.skip_indexes.items() if "inverted" in kinds]
        ss = [marshal_segment(s, self.m, skip_inverted=skip) for s in self.segs]
        qs = [marshal_query(s, q, self.m) for s in self.segs]
        n = len(self.segs)
        self.seg_ptrs = (C.POINTER(OrcSegment) * n)(*[C.pointer(x) for x in ss])
        self.q_ptrs = (C.POINTER(OrcQuery) * n)(*[C.pointer(x) for x in qs])
        self.out = (C.c_void_p * n)()


def execute_batch(prep: "PreparedBatch", threads: int) -> List["OracleResult"]:
    """All segments of the query on `threads` native worker threads (pthreads inside liboracle.so: no interpreter in the
    loop), like one GroupByCombineOperator pass before the merge."""
    l = lib()
    n = len(prep.segs)
    failed = l.orc_execute_batch(prep.seg_ptrs, prep.q_ptrs, n, threads, prep.out)
    try:
        if failed:
            raise RuntimeError("oracle: " + l.orc_last_error().decode())
        return [OracleResult(s, prep.q, prep.out[i]) for i, s in enumerate(prep.segs)]
    finally:
        for i in range(n):
            if prep.out[i]:
                l.orc_result_free(prep.out[i])
                prep.out[i] = None


def execute_combined(prep: "PreparedBatch", threads: int):
    """One GroupByCombineOperator-style pass entirely in native code: the segments on `threads` pooled worker threads, each
    folding its results into an IndexedTable keyed by the decoded group key, tables merged at the end (orc_execute_combined).
    Returns (keys[n, nG] int64 -- FLOAT / DOUBLE keys as bit patterns --, doubles[n, nA], longs[n, nA]), or None when the query
    needs the Python merge (DISTINCTCOUNT, STRING keys)."""
    l = lib()
    kp, dp, lp = C.POINTER(C.c_int64)(), C.POINTER(C.c_double)(), C.POINTER(C.c_int64)()
    n = l.orc_execute_combined(prep.seg_ptrs, prep.q_ptrs, len(prep.segs), threads, C.byref(kp), C.byref(dp), C.byref(lp))
    if n < 0:
        return None
    nG, nA = len(prep.q.group_by), len(prep.q.aggregations)
    try:
        keys = np.ctypeslib.as_array(kp, shape=(max(n, 1) * max(nG, 1),))[:n * nG].reshape(n, nG).copy()
        dbl = np.ctypeslib.as_array(dp, shape=(max(n, 1) * nA,))[:n * nA].reshape(n, nA).copy()
        lng = np.ctypeslib.as_array(lp, shape=(max(n, 1) * nA,))[:n * nA].reshape(n, nA).copy()
    finally:
        for ptr in (kp, dp, lp):
            l.orc_free(ptr)
    return keys, dbl, lng


def filter_doc_ids(seg, q):
    m = _Marshalled()
    skip = [c for c, kinds in q.skip_indexes.items() if "inverted" in kinds]
    s = marshal_segment(seg, m, skip_inverted=skip)
    oq = marshal_query(seg, q, m)
    out = C.POINTER(C.c_int32)()
    entries = C.c_int64(0)
    n = lib().orc_filter_doc_ids(C.byref(s), C.byref(oq), C.byref(out), C.byref(entries))
    if n < 0:
        raise RuntimeError("oracle: " + lib().orc_last_error().decode())
    docs = np.ctypeslib.as_array(out, shape=(max(n, 1),))[:n].copy()
    lib().orc_free(out)
    return docs, entries.value


def combine(results: List[OracleResult]) -> Dict[tuple, list]:
    """Cross-segment merge by decoded key (GroupByCombineOperator.java:132-147, IndexedTable.java:99-125):
    SUM add, MIN min, MAX max, COUNT add, AVG (sum,count) add, DISTINCTCOUNT set union (by value)."""
    table: Dict[tuple, list] = {}
    for r in results:
        q = r.query
        keys = r.decoded_keys() if q.group_by else [()]
        dvals = []
        for a, agg in enumerate(q.aggregations):
            if int(agg.op) == 5 and r.segment.columns[agg.column].has_dictionary:
                dvals.append(r.segment.columns[agg.column].dictionary_values())
            else:
                dvals.append(None)      # (DISTINCTCOUNT on a raw column: the sets hold the value bits themselves)
        nh = getattr(q, "null_handling", False)     # longs hold the inputs every function saw; 0 = SQL NULL (merge: SumAggregationFunction.java:222-233)
        for g, key in enumerate(keys):
            row = []
            for a, agg in enumerate(q.aggregations):
                op = int(agg.op)
                if op == 0:
                    row.append(int(r.longs[a][g]))
                elif op in (1, 2, 3):
                    row.append(None if nh and int(r.longs[a][g]) == 0 else float(r.doubles[a][g]))
                elif op == 4:
                    row.append((float(r.doubles[a][g]), int(r.longs[a][g])))
                else:
                    off, ids = r.distinct[a]
                    row.append(set((dvals[a][ids[off[g]:off[g + 1]]] if dvals[a] is not None else ids[off[g]:off[g + 1]]).tolist()))
            cur = table.get(key)
            if cur is None:
                table[key] = row
                continue
            for a, agg in enumerate(q.aggregations):
                op = int(agg.op)
                if cur[a] is None or row[a] is None:
                    cur[a] = row[a] if cur[a] is None else cur[a]
                elif op in (0, 1):
                    cur[a] = cur[a] + row[a]
                elif op == 2:
                    cur[a] = min(cur[a], row[a])
                elif op == 3:
                    cur[a] = max(cur[a], row[a])
                elif op == 4:
                    cur[a] = (cur[a][0] + row[a][0], cur[a][1] + row[a][1])
                else:
                    cur[a] = cur[a] | row[a]
    if results and getattr(results[0].query, "null_handling", False):
        for row in table.values():
            for a, agg in enumerate(results[0].query.aggregations):
                if int(agg.op) == 4 and row[a][1] == 0:
                    row[a] = None
    return table


def combine_numeric(results: List[OracleResult]):
    """Vectorised cross-segment merge for numeric group keys and COUNT/SUM/MIN/MAX/AVG (same semantics as
    combine(); used where the merge itself is timed).  Returns (keys[n, nG], [per-aggregation arrays])."""
    q = results[0].query
    cols = [results[0].segment.columns[c] for c in q.group_by]
    if any(int(a.op) == 5 for a in q.aggregations) or any(c.data_type.name == "STRING" for c in cols):
        return combine(results)
    key_blocks = []
    for r in results:
        if not q.group_by:
            key_blocks.append(np.zeros((1, 0), dtype=np.int64))
            continue
        blk = np.empty((r.num_groups, len(q.group_by)), dtype=np.float64)
        for j, cname in enumerate(q.group_by):
            c = r.segment.columns[cname]
            if c.has_dictionary:
                blk[:, j] = c.dictionary_values()[r.group_keys[:, j]]
            elif c.data_type.name in ("FLOAT", "DOUBLE"):
                blk[:, j] = r.group_keys[:, j].view(np.float64)
            else:
                blk[:, j] = r.group_keys[:, j]
        key_blocks.append(blk)
    allk = np.concatenate(key_blocks, axis=0)
    if allk.shape[1] == 0:
        uniq, inv = np.zeros((1, 0)), np.zeros(allk.shape[0], dtype=np.int64)
    else:
        uniq, inv = np.unique(allk, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
    n = uniq.shape[0]
    out = []
    for a, agg in enumerate(q.aggregations):
        op = int(agg.op)
        d = np.concatenate([r.doubles[a] for r in results])
        l = np.concatenate([r.longs[a] for r in results])
        if op == 0:
            acc = np.zeros(n, dtype=np.int64); np.add.at(acc, inv, l); out.append(acc)
        elif op == 1:
            acc = np.zeros(n); np.add.at(acc, inv, d); out.append(acc)
        elif op == 2:
            acc = np.full(n, np.inf); np.minimum.at(acc, inv, d); out.append(acc)
        elif op == 3:
            acc = np.full(n, -np.inf); np.maximum.at(acc, inv, d); out.append(acc)
        else:
            acc = np.zeros(n); np.add.at(acc, inv, d)
            cnt = np.zeros(n, dtype=np.int64); np.add.at(cnt, inv, l); out.append((acc, cnt))
    return uniq, out
