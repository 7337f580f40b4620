"""The HBM segment cache (-m gpu): with hbm_cache_bytes set, pb_init bounds the bytes staged per device; after staging, a
call drops the least recently used segments no query is using (enforce_cache_limit), a segment keeps at most 4 row groups
(row_group_for drops the least recently used one), and both kinds of drop bump the segment's epoch, which retires every
parked plan and CUDA graph that points into the freed memory.  A mistake here does not crash: the kernels read a re-staged
or re-used pool block and return plausible numbers.  So every call below is held to the exact reference (tests/reference.py),
per segment and with PB_Q_COMBINE, and after every call the cache's own bookkeeping is checked against a model kept here:

* the staged bytes pb_cache_stats reports equal the sum of pb_segment_device_bytes over the live segments;
* the segments a call dropped are exactly a least-recently-used prefix of the staged segments the call did not touch and
  no deferred result pins, and the eviction counter grew by their number;
* afterwards the staged bytes are within the limit, or nothing the call did not touch is left to drop.

A later pb_init can change the limit but never set it back to 0, so the scenarios run in one child process (this module
again, under PB_SEGMENT_CACHE_CHILD=1); the suite's own process never evicts.  Each scenario stages its segments under an
unbounded limit, reads their sizes, and then sets its limit from them: no byte count is written down here.  Whether the
first call after staging is parked depends on whether its copies had finished; no test asserts on it."""
import os
import re
import subprocess
import sys
from contextlib import contextmanager

import numpy as np
import pytest

from pinot_b200 import native
from pinot_b200.query import parse_sql
from pinot_b200.segment_writer import DataType, build_column, make_segment, with_nulls
from tests import fuzz_gen
from tests.reference import Col, assert_matches_reference, concat, evaluate_sql, reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD_ENV = "PB_SEGMENT_CACHE_CHILD"
IN_CHILD = os.environ.get(CHILD_ENV) == "1"
CHILD_TIMEOUT_S = 900
UNBOUNDED = 2 ** 62
PB_ERR_INVALID = -1                  # include/pinot_b200.h
NGL = "SET numGroupsLimit = 100000000; "

pytestmark = pytest.mark.gpu


def child(f):
    """a scenario: runs only in the child process"""
    f.in_child = True
    return pytest.mark.skipif(not IN_CHILD, reason=f"runs in the child process of test_segment_cache_scenarios ({CHILD_ENV}=1)")(f)


# ---- the parent process ----

@pytest.mark.skipif(IN_CHILD, reason="the parent's test")
def test_segment_cache_scenarios():
    """every scenario below, in one child process: its limits never reach the rest of the suite.  The child runs under
    the default knobs (the library reads most of them once per process)."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("PB_") or k == "PB_LIB_PATH"}
    env.update({CHILD_ENV: "1", "PYTHONDONTWRITEBYTECODE": "1"})
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)]
    try:
        p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=CHILD_TIMEOUT_S)
        rc, out = p.returncode, (p.stdout + p.stderr)[-8000:]
    except subprocess.TimeoutExpired as e:
        rc, out = -1, f"timed out after {CHILD_TIMEOUT_S} s\n" + str(e.stdout or "")[-6000:]
    assert rc == 0, out
    n = sum(1 for k, f in globals().items() if k.startswith("test_") and getattr(f, "in_child", False))
    assert re.search(rf"\b{n} passed, 2 skipped\b", out), f"expected {n} scenarios to pass:\n{out}"


@pytest.mark.skipif(IN_CHILD, reason="the parent's test")
def test_the_suite_process_never_evicts():
    native.init()
    assert native.cache_stats()[1] == 0, native.cache_stats()


# ---- tables ----

def fuzz_table(n_segs, docs=30_000, seed=5):
    """fuzz_gen's columns (dictionaries of several widths, sorted, inverted, var-length STRING, raw, LZ4 / Snappy raw) plus
    `nul`, an INT dictionary column with a null-value vector"""
    segs, srcs, _ = fuzz_gen.make_tables(seed, sizes=[docs + 7 * i for i in range(n_segs)])
    for si, (seg, src) in enumerate(zip(segs, srcs)):
        r = np.random.default_rng([seed, 900 + si])
        v = r.integers(0, 50, seg.num_docs)
        nulls = r.random(seg.num_docs) < 0.3
        seg.columns["nul"] = with_nulls(build_column("nul", DataType.INT, np.where(nulls, -(2 ** 31), v).astype(np.int32)), nulls)
        src["nul"] = Col(np.where(nulls, -(2 ** 31), v).astype(np.int64), DataType.INT, True, nulls)
    return segs, srcs


# every query reads a column of some kind: a sorted and an inverted leaf, IS NULL over a null-value vector, a
# chunk-compressed raw input, var-length STRING keys, DISTINCTCOUNT
QUERIES = [
    "SELECT k3, COUNT(*), SUM(mint), MAX(mdbl) FROM t WHERE fsort < 20 GROUP BY k3 LIMIT 1000",
    "SELECT k2, COUNT(*), MIN(mlong), SUM(fu) FROM t WHERE finv IN (3, 17, 150, 199) OR finv = 40 GROUP BY k2 LIMIT 1000",
    "SELECT k3, COUNT(*), SUM(mlong), MIN(mflt) FROM t WHERE nul IS NULL GROUP BY k3 LIMIT 1000",
    "SELECT k3, SUM(rz), MIN(rz), MAX(rz), COUNT(*) FROM t WHERE fu < 1200 GROUP BY k3 LIMIT 1000",
    "SELECT kstr, COUNT(*), AVG(mflt), MAX(rint) FROM t WHERE k2 = 10 GROUP BY kstr LIMIT 1000",
    "SELECT k2, DISTINCTCOUNT(mint), DISTINCTCOUNT(kstr), COUNT(*) FROM t WHERE nul IS NOT NULL AND fsort >= 10 GROUP BY k2 LIMIT 1000",
]


class Cache:
    """The live segments of one scenario and the model of what the cache must do after each call"""

    def __init__(self, segs, srcs):
        native.init(hbm_cache_bytes=UNBOUNDED)
        self.segs, self.srcs = segs, srcs
        self.staged = [native.StagedSegment(s) for s in segs]
        self.groups = []
        self.last = {}                       # segment index -> (call number, position in the call): its last use
        self.calls = 0
        self.limit = UNBOUNDED
        self.dropped = set()                 # segments the cache has dropped at least once
        self.restaged = set()                # query texts that staged columns again on such a segment
        self.kept = []                       # results handed out alive: freed before their groups
        self.deferred = []                   # (result, segments) of deferred results not finalized yet: they pin their segments

    def group(self, idx):
        g = native.SegmentGroup([self.staged[i] for i in idx])
        self.groups.append(g)
        return g

    def set_limit(self, limit):
        self.limit = limit
        native.init(hbm_cache_bytes=limit)

    def bytes(self):
        return [s.device_bytes() for s in self.staged]

    def check_accounting(self, what):
        staged = native.cache_stats()[0]
        total = sum(self.bytes())
        assert staged == total, f"{what}: the cache reports {staged} staged bytes, the live segments hold {total}"

    def call(self, g, idx, sql, flags, keep=False, check=True):
        """one execute on group g (segments idx), checked against the reference and the model; returns the Result (freed
        unless keep) and its handle"""
        before, ev0 = self.bytes(), native.cache_stats()[1]
        q = parse_sql(sql)
        res = native.execute(g, q, flags)
        self.calls += 1
        what = f"call {self.calls} segments {list(idx)} flags {flags}: {sql}"
        after, (staged, ev1) = self.bytes(), native.cache_stats()
        # the model: touched segments are never dropped; the dropped ones are the least recently used of the others
        for i in idx:
            assert after[i] > 0, f"{what}: segment {i}, used by the call, holds no bytes"
            if before[i] < after[i] and i in self.dropped:
                self.restaged.add(sql)
        pinned = self.pinned()
        untouched = sorted((i for i in range(len(self.staged)) if i not in idx and i not in pinned and before[i] > 0),
                           key=lambda i: self.last[i])
        dropped = [i for i in untouched if after[i] == 0]
        assert dropped == untouched[:len(dropped)], \
            f"{what}: dropped {dropped}, the least recently used first were {untouched} (last uses {[self.last[i] for i in untouched]})"
        assert ev1 - ev0 == len(dropped), f"{what}: {ev1 - ev0} evictions counted, {len(dropped)} segments dropped"
        self.dropped.update(dropped)
        assert staged == sum(after), f"{what}: the cache reports {staged} staged bytes, the live segments hold {sum(after)}"
        assert staged <= self.limit or all(after[i] == 0 for i in untouched), \
            f"{what}: {staged} bytes staged > limit {self.limit} with segments {[i for i in untouched if after[i]]} left to drop"
        for pos, i in enumerate(idx):
            self.last[i] = (self.calls, pos)
        if check and not flags & native.PB_Q_DEFER_FINALIZE:
            self.check_result(res, idx, q, flags, what)
        h = res._rh.value
        if keep:
            self.kept.append(res)
            if flags & native.PB_Q_DEFER_FINALIZE:
                self.deferred.append((res, list(idx)))
        else:
            res.free()
        return res, h

    def check_result(self, res, idx, q, flags, what):
        if flags & native.PB_Q_COMBINE:
            parts = [(res.tables[0], concat([self.srcs[i] for i in idx]), sum(self.segs[i].num_docs for i in idx))]
        else:
            parts = [(t, self.srcs[i], self.segs[i].num_docs) for t, i in zip(res.tables, idx)]
        assert len(parts) == (1 if flags & native.PB_Q_COMBINE else len(idx)), what
        for t, src, n in parts:
            assert_matches_reference(t.rows(), reference(src, q), q, what)
            assert t.stats["num_docs_scanned"] == int(evaluate_sql(src, q.filter).sum()), what
            assert t.stats["num_total_docs"] == n, what

    def both(self, g, idx, sql):
        """per segment, then combined"""
        self.call(g, idx, sql, 0)
        self.call(g, idx, sql, native.PB_Q_COMBINE)

    def pinned(self):
        return {i for _, idx in self.deferred for i in idx}

    def finalize(self, res):
        res.finalize()
        self.deferred = [(r, idx) for r, idx in self.deferred if r is not res]

    def release(self):
        for r in self.kept:
            r.free()
        self.kept, self.deferred = [], []
        for g in self.groups:
            g.release()
        for s in self.staged:
            s.release()
        native.init(hbm_cache_bytes=UNBOUNDED)
        assert native.cache_stats()[0] == 0, native.cache_stats()


@contextmanager
def cache(n_segs, **kw):
    c = Cache(*fuzz_table(n_segs, **kw))
    try:
        yield c
    finally:
        c.release()


def _replayed(res):
    """the call ran a parked plan: its planning stages did not run (pb_result_host_timing slots 1 and 2)"""
    t = res.host_timing_us()
    return t[1] == 0 and t[2] == 0


def run_until_replay(c, g, idx, sql, flags, max_calls=4):
    """call until the handle of a call repeats that of the call before and the call ran a parked plan; returns it"""
    prev = None
    for _ in range(max_calls):
        res, h = c.call(g, idx, sql, flags, keep=True)
        rep = _replayed(res)
        res.free()
        if h == prev and rep:
            return h
        prev = h
    raise AssertionError(f"no replay in {max_calls} calls: {sql}")


def visit(c, g, idx, rot=0, both=False):
    """every query kind on one group, starting with QUERIES[rot]"""
    for j in range(len(QUERIES)):
        sql = QUERIES[(rot + j) % len(QUERIES)]
        if both:
            c.both(g, idx, sql)
        else:
            c.call(g, idx, sql, native.PB_Q_COMBINE)


def warm(c, groups):
    """stage what the scenario reads under the unbounded limit, and return each segment's size then: a visit leaves a
    segment about that large again"""
    for g, idx in groups:
        visit(c, g, idx)
    return c.bytes()


def evict(c, target, singles, max_visits=8):
    """visit the other one-segment groups in turn until segment `target` is dropped"""
    others = [s for s in singles if s[1][0] != target]
    for v in range(max_visits):
        if c.bytes()[target] == 0:
            return
        visit(c, *others[v % len(others)], rot=v)
    assert c.bytes()[target] == 0, f"segment {target} was not evicted in {max_visits} visits"


# ---- scenarios (child process) ----

@child
def test_lru_eviction_and_restaging():
    """five one-segment groups and one over all of them, a limit of about two and a half segments, a script that moves
    through every query kind: every query on a segment just dropped re-stages it (sorted-to-packed rebuild, chunk re-decode,
    inverted re-expansion) and equals the reference"""
    with cache(5) as c:
        singles = [(c.group([i]), [i]) for i in range(5)]
        everything = (c.group(list(range(5))), list(range(5)))
        full = warm(c, singles)
        c.check_accounting("warm")
        c.set_limit(int(2.5 * np.mean(full)))
        order = [0, 1, 2, 3, 4, 0, 2, 4, 1, 3]
        for step, si in enumerate(order):
            visit(c, *singles[si], rot=step, both=True)
            if step % 5 == 4:
                c.both(*everything, QUERIES[step % len(QUERIES)])
        assert native.cache_stats()[1] >= 8, native.cache_stats()
        assert c.restaged >= set(QUERIES), f"queries that never re-staged a segment: {set(QUERIES) - c.restaged}"


@child
def test_limit_below_one_segment():
    """every call re-stages its segment and is still exact; the segment a call uses is never dropped"""
    with cache(3, docs=12_000) as c:
        singles = [(c.group([i]), [i]) for i in range(3)]
        full = warm(c, singles)
        assert min(full) > 1
        c.set_limit(1)
        for step in range(12):
            g, idx = singles[step % 3]
            before = c.bytes()
            assert step == 0 or before[idx[0]] == 0, f"step {step}: segment {idx[0]} still staged under a limit below one segment"
            c.call(g, idx, QUERIES[step % len(QUERIES)], native.PB_Q_COMBINE if step % 2 else 0)
            assert sum(b > 0 for b in c.bytes()) == 1, c.bytes()


@child
def test_pinned_segments_survive():
    """a deferred combined result pins its group's segments: calls on other groups that push the staged bytes over the
    limit drop only the others, and the held result then finalizes to the reference"""
    with cache(5) as c:
        singles = [(c.group([i]), [i]) for i in range(5)]
        a_idx = [0, 1]
        a = c.group(a_idx)
        full = warm(c, singles)
        c.set_limit(int(2.5 * np.mean(full)))
        sql = NGL + QUERIES[3]
        held, _ = c.call(a, a_idx, sql, native.PB_Q_DEFER_FINALIZE | native.PB_Q_COMBINE, keep=True)
        kept = c.bytes()
        ev0 = native.cache_stats()[1]
        for step, si in enumerate([2, 3, 4, 2, 3, 4]):
            visit(c, *singles[si], rot=step)
            assert c.bytes()[:2] == kept[:2], f"step {step}: the pinned segments lost bytes: {kept[:2]} -> {c.bytes()[:2]}"
        assert native.cache_stats()[1] > ev0, "no call had to evict"
        c.finalize(held)
        q = parse_sql(sql)
        c.check_result(held, a_idx, q, native.PB_Q_COMBINE, "held deferred result")
        held.free()


@child
def test_eviction_retires_parked_plans():
    """a plan parked on a segment that is then evicted is never replayed: the next call plans afresh (a new handle while
    the parked one is still alive), equals the reference, and within two more calls replays its own plan, exactly"""
    with cache(5) as c:
        singles = [(c.group([i]), [i]) for i in range(5)]
        full = warm(c, singles)
        c.set_limit(int(2.5 * np.mean(full)))
        for sql in (QUERIES[0], QUERIES[3], QUERIES[5]):
            g, idx = singles[0]
            parked = run_until_replay(c, g, idx, sql, native.PB_Q_COMBINE)
            evict(c, 0, singles)
            res, h = c.call(g, idx, sql, native.PB_Q_COMBINE, keep=True)
            assert h != parked and not _replayed(res), f"the plan parked before the eviction was replayed: {sql}"
            res.free()
            prev, replayed = h, False
            for _ in range(2):
                res, h = c.call(g, idx, sql, native.PB_Q_COMBINE, keep=True)
                replayed = h == prev and _replayed(res)
                res.free()
                if replayed:
                    break
                prev = h
            assert replayed, f"no replay within two calls after re-staging: {sql}"


# row-group shapes: (keys, aggregations, row bits); no shape's (column, form) set lies inside another's, so each builds
# its own row group.  Bits: k2 1, k3 2, kstr <= 6, fsort <= 6, finv 8 (dictIds); mint, mflt, fu 32, mlong, mdbl 64 (values).
SHAPES = [
    ("k3", "SUM(mint), COUNT(*)", 2 + 32),
    ("k2", "SUM(mlong), MAX(mlong)", 1 + 64),
    ("kstr", "MIN(mdbl), MAX(mlong)", 6 + 64 + 64),
    ("finv", "SUM(mflt), MIN(mflt)", 8 + 32),
    ("k3, k2", "SUM(fu), MAX(fu)", 2 + 1 + 32),
    ("fsort", "MAX(mdbl), AVG(mdbl)", 6 + 64),
]


def _shape_sql(shape):
    keys, aggs, _ = shape
    return f"{NGL}SELECT {keys}, {aggs} FROM t WHERE fu < 700 GROUP BY {keys} LIMIT 100000"      # about 35 % of the docs


def _rw(bits):
    return 2 if bits <= 64 else 4 if bits <= 128 else 8


@child
def test_row_group_replacement():
    """five shapes over one segment, each through its own group, cycled twice: the fifth shape drops the least recently
    used row group, which retires every plan parked on the segment; every call runs pb_agg_rows_kernel at the row width
    the shape asks for and equals the reference.  Then, with a deferred result holding the segment, a call that needs a
    row group the segment does not have gets none: it runs without one, exactly, and the held result finalizes exactly."""
    with cache(1, docs=40_000) as c:
        seg = [0]
        for keys, _, bits in SHAPES:
            for k in keys.split(", "):
                width = {"k2": 1, "k3": 2, "kstr": 6, "fsort": 6, "finv": 8}[k]
                assert c.segs[0].columns[k].bits_per_element <= width, (k, c.segs[0].columns[k].bits_per_element)
        groups = [c.group(seg) for _ in SHAPES]
        resident = []                          # shape indices whose row group the segment holds, least recently used first
        parked = {}                            # shape -> handle of its parked plan (alive: its group keeps at most 8)
        epoch = 0
        parked_epoch = {}
        for cycle in range(2):
            for si in range(5):
                sql = _shape_sql(SHAPES[si])
                if si in resident:
                    resident.remove(si)
                elif len(resident) == 4:
                    resident.pop(0)
                    epoch += 1
                resident.append(si)
                if si in parked:
                    res, h = c.call(groups[si], seg, sql, native.PB_Q_COMBINE, keep=True)
                    if parked_epoch[si] != epoch:
                        assert h != parked[si] and not _replayed(res), f"cycle {cycle} shape {si}: a retired plan was replayed"
                    res.free()
                for run in range(3):
                    res, h = c.call(groups[si], seg, sql, native.PB_Q_COMBINE, keep=True)
                    pi = res.plan_info
                    assert pi["agg_kernel"] == 3 and pi["rows_rw"] == _rw(SHAPES[si][2]), (cycle, si, run, pi)
                    if run == 2:
                        parked[si], parked_epoch[si] = h, epoch
                    res.free()
                c.call(groups[si], seg, sql, 0)
        assert epoch >= 2, epoch
        # a deferred result on a resident shape pins the segment: a sixth shape gets no row group
        hold_si = resident[-1]
        hsql = _shape_sql(SHAPES[hold_si])
        held, _ = c.call(groups[hold_si], seg, hsql, native.PB_Q_DEFER_FINALIZE | native.PB_Q_COMBINE, keep=True)
        assert held.plan_info["agg_kernel"] == 3, held.plan_info
        sixth = c.group(seg)
        res, _ = c.call(sixth, seg, _shape_sql(SHAPES[5]), native.PB_Q_COMBINE, keep=True)
        pi = res.plan_info
        assert pi["agg_kernel"] != 3 and pi["rows_rw"] == 0, f"planned onto a row group while the segment was held: {pi}"
        res.free()
        c.finalize(held)
        c.check_result(held, seg, parse_sql(hsql), native.PB_Q_COMBINE, "held deferred result")
        held.free()
        # released: the sixth shape, planned afresh (its own plan without a row group may be parked), replaces a row group
        res, _ = c.call(c.group(seg), seg, _shape_sql(SHAPES[5]), native.PB_Q_COMBINE, keep=True)
        assert res.plan_info["agg_kernel"] == 3 and res.plan_info["rows_rw"] == _rw(SHAPES[5][2]), res.plan_info
        res.free()


@child
def test_global_dictionary_change_retires_parked_plans():
    """after set_global_dictionary with a wider union, the parked combined plan is not replayed: its group keys follow
    the new global dictIds and the values equal the reference"""
    with cache(3, docs=20_000) as c:
        idx = [0, 1, 2]
        g = c.group(idx)
        sql = QUERIES[0]
        parked = run_until_replay(c, g, idx, sql, native.PB_Q_COMBINE)
        wider = np.array([-9, -5, -1, 0, 3, 7, 11], dtype=np.int32)
        assert set(np.unique(np.concatenate([c.srcs[i]["k3"].values for i in idx]))) <= set(wider.tolist())
        g.set_global_dictionary("k3", wider.view(np.uint8).reshape(-1, 4))
        for run in range(3):
            res, h = c.call(g, idx, sql, native.PB_Q_COMBINE, keep=True)
            if run == 0:
                assert h != parked and not _replayed(res), "the plan parked before the dictionary change was replayed"
            t = res.tables[0]
            ids, vals = t.key_dict_ids[0], t.key_values[0]
            assert (wider[ids] == vals).all(), f"run {run}: group keys do not follow the new global dictIds: {ids} {vals}"
            res.free()


@child
def test_a_held_result_outlives_the_plan_limit():
    """a group keeps at most 8 plans and destroys the oldest idle one: a result held while ten other queries park plans
    stays intact and exact, and its query afterwards is replayed or planned again, never corrupted"""
    with cache(2, docs=20_000) as c:
        idx = [0, 1]
        g = c.group(idx)
        sql = QUERIES[1]
        c.call(g, idx, sql, native.PB_Q_COMBINE)
        held, _ = c.call(g, idx, sql, native.PB_Q_COMBINE, keep=True)
        snapshot = {k: list(v) for k, v in held.tables[0].rows().items()}
        for i in range(10):
            other = f"SELECT k3, COUNT(*), SUM(mint) FROM t WHERE fu < {200 + 90 * i} GROUP BY k3 LIMIT 1000"
            for _ in range(2):
                c.call(g, idx, other, native.PB_Q_COMBINE)
        c.check_result(held, idx, parse_sql(sql), native.PB_Q_COMBINE, "held result")
        assert {k: list(v) for k, v in held.tables[0].rows().items()} == snapshot
        held.free()
        for _ in range(3):
            c.call(g, idx, sql, native.PB_Q_COMBINE)


@child
def test_cold_reads_after_eviction():
    """a segment whose forward indexes are page-locked is evicted; a PB_Q_GATHER_IN_PLACE call then reads columns where
    they lie (PB_IN_PLACE_COST=0), exactly; the first normal call on the same group afterwards is planned afresh (in-place
    calls are not cached), and the next one replays that call's plan or plans again: both exact"""
    c = Cache(*fuzz_table(4, docs=20_000))
    bufs = [c.segs[0].columns[n].forward_index for n in ("k3", "mint", "rdbl", "fu")]
    for b in bufs:
        native.host_register(b)
    try:
        singles = [(c.group([i]), [i]) for i in range(4)]
        full = warm(c, singles)
        c.set_limit(int(1.5 * np.mean(full)))
        evict(c, 0, singles)
        sql = "SELECT k3, COUNT(*), SUM(mint), MAX(rdbl) FROM t WHERE fu < 300 GROUP BY k3 LIMIT 1000"
        os.environ["PB_IN_PLACE_COST"] = "0"
        try:
            res, _ = c.call(*singles[0], sql, native.PB_Q_GATHER_IN_PLACE | native.PB_Q_COMBINE, keep=True)
        finally:
            del os.environ["PB_IN_PLACE_COST"]
        assert res.in_place_columns > 0, res.in_place_columns
        res.free()
        res, first = c.call(*singles[0], sql, native.PB_Q_COMBINE, keep=True)
        assert res.in_place_columns == 0 and not _replayed(res), "the first normal call replayed a plan"
        res.free()
        # (whether the first call was parked depends on whether its copies had finished when it was planned)
        res, h = c.call(*singles[0], sql, native.PB_Q_COMBINE, keep=True)
        assert res.in_place_columns == 0
        assert not _replayed(res) or h == first, "the second normal call replayed a plan other than the first call's"
        res.free()
    finally:
        c.release()                # the segments go before their host buffers are unregistered
        for b in bufs:
            native.host_unregister(b)


def _bad_segment():
    """a dictionary key `k` and `z`, a raw LONG column whose first LZ4 chunk is malformed (test_gpu_index_decoding)"""
    import pyarrow as pa
    from tests.test_gpu_index_decoding import _malformed
    rng = np.random.default_rng(4601)
    n, dpc = 5000, 1000
    k = rng.integers(0, 7, n)
    v = rng.integers(-100, 100, n)
    z = np.cumsum(rng.integers(0, 5, n)).astype(np.int64)
    raw0 = z[:dpc].astype(">i8").tobytes()
    bad = _malformed("lz4 offset past the output", raw0)
    zcol = build_column("z", DataType.LONG, z, dictionary=False, raw_compression="LZ4", raw_docs_per_chunk=dpc,
                        raw_block=lambda raw: bad if raw == raw0 else pa.Codec("lz4_raw").compress(raw, asbytes=True))
    seg = make_segment("refused", [build_column("k", DataType.INT, k.astype(np.int32)), build_column("v", DataType.INT, v.astype(np.int32)), zcol])
    return seg, {"k": Col(k, DataType.INT), "v": Col(v, DataType.INT)}


@child
def test_refused_call_keeps_the_accounting():
    """a call that stages its group key and is then refused on a malformed chunk (PB_ERR_INVALID) leaves the key in HBM:
    the cache counts it, and a later eviction and a valid query on that segment are exact"""
    segs, srcs = fuzz_table(2, docs=10_000)
    bad, bad_src = _bad_segment()
    c = Cache(segs + [bad], srcs + [bad_src])
    try:
        singles = [(c.group([i]), [i]) for i in range(3)]
        full = warm(c, singles[:2])
        c.set_limit(int(1.5 * max(full)))
        with pytest.raises(native.PinotB200Error) as e:
            native.execute(singles[2][0], parse_sql("SELECT k, SUM(z) FROM t GROUP BY k LIMIT 100"), 0)
        assert e.value.code == PB_ERR_INVALID and "do not decode" in str(e.value), str(e.value)
        assert c.bytes()[2] > 0, "the refused call staged nothing"
        c.check_accounting("after the refused call")
        c.last[2] = (c.calls, 0)
        good = "SELECT k, COUNT(*), SUM(v), MIN(v) FROM t WHERE v > -50 GROUP BY k LIMIT 100"
        c.both(*singles[2], good)
        c.set_limit(1)
        c.call(*singles[0], QUERIES[2], 0)
        assert c.bytes()[2] == 0, "the segment of the refused call was not evicted"
        c.both(*singles[2], good)
        c.check_accounting("end")
    finally:
        c.release()
