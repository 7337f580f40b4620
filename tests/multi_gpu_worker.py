"""Worker of tests/test_gpu_multi.py (and usable by hand on a multi-GPU box):

    python tests/multi_gpu_worker.py ranks <rank> <world> <exchange_dir>     one process per GPU: NCCL inside the library
    python tests/multi_gpu_worker.py devices <n_devices>                      one process driving n GPUs: NVLink peer merge

Every rank / device owns its own segments (different dictionaries per segment); the merged result of every query must be
exactly what the oracle's cross-segment merge (oracle.combine) gives over ALL segments of ALL ranks.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

try:
    # The library dlopens whichever libnccl the process already maps before it falls back to the system one (pb_comm_init):
    # with torch imported that is the copy torch ships -- the one bench.py and a torchrun deployment run on.  (Open: without
    # it, on the system's NCCL, 4 ranks once tripped the layout-fingerprint check of the merged block; cause not found.)
    import torch  # noqa: E402,F401
except Exception:  # pragma: no cover
    pass

from oracle import oracle  # noqa: E402
from pinot_b200 import datagen, native  # noqa: E402
from pinot_b200.query import parse_sql  # noqa: E402
from tests.parity import assert_rows_equal, combined_rows  # noqa: E402

COLS = ["c1", "c2", "c3", "d0", "d1", "d2", "m0", "m1", "m2", "x0", "k0"]
SEGS_PER_PART = 2
DOCS = 60_000


def segment(i):
    # odd segments draw their own dimension dictionaries: the local -> global dictId remap matters
    return datagen.make_segment_synth(i, DOCS + 1000 * i, columns=COLS, vary_dim_dictionaries=(i % 2 == 1))


def queries(segs):
    d2 = segs[0].columns["c2"].dictionary_values()
    d3 = segs[0].columns["c3"].dictionary_values()
    k2, k3 = int(d2[len(d2) // 2]), int(d3[len(d3) // 3])
    return [
        ("dense", f"SELECT d0, d1, d2, SUM(m0), COUNT(*), MIN(m1), MAX(m2), AVG(m0) FROM t WHERE c2 < {k2} GROUP BY d0, d1, d2 LIMIT 100000", True),
        ("dense double sum", f"SELECT d1, SUM(x0), MAX(x0) FROM t WHERE c3 > {k3} GROUP BY d1 LIMIT 100000", False),
        ("distinctcount", f"SELECT d0, DISTINCTCOUNT(c3), DISTINCTCOUNT(c1), SUM(m1) FROM t WHERE c2 < {k2} GROUP BY d0 LIMIT 100000", True),
        ("filtered aggregation", f"SELECT d1, SUM(m0) FILTER(WHERE c3 < {k3}), COUNT(*) FILTER(WHERE c3 < {k3}), MAX(m2), COUNT(*) FROM t "
                                 f"WHERE c2 < {k2} GROUP BY d1 LIMIT 100000", True),
        ("keyless", f"SELECT COUNT(*), SUM(m0), MIN(m1), MAX(m2), DISTINCTCOUNT(c3) FROM t WHERE c2 >= {k2}", True),
        ("match all", "SELECT d2, COUNT(*), SUM(m2) FROM t GROUP BY d2 LIMIT 100000", True),
    ]


def expected(all_segs, q):
    orc = [oracle.execute(s, q) for s in all_segs]
    return combined_rows(oracle.combine(orc), q), orc


def check(name, res, exp, orc, q, exact, n_segments_total):
    assert len(res.tables) == 1, name
    t = res.tables[0]
    assert_rows_equal(t.rows(), exp, q, exact_float=exact, what=name)
    st = t.stats
    assert st["num_docs_scanned"] == sum(o.stats["num_docs_scanned"] for o in orc), (name, st)
    assert st["num_entries_scanned_post_filter"] == sum(o.stats["num_entries_scanned_post_filter"] for o in orc), (name, st)
    assert st["num_total_docs"] == sum(o.stats["num_total_docs"] for o in orc), (name, st)
    assert st["num_segments"] == n_segments_total, (name, st)


def run_ranks(rank, world, xdir):
    from pinot_b200.distributed import FileExchange, agree_global_dictionaries, dictionary_columns, init_comm
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    native.init(rank)                                   # this process drives CUDA device `rank`
    ex = FileExchange(xdir, rank, world)
    init_comm(ex)
    assert native.comm_info() == (True, world, rank)
    all_segs = [segment(i) for i in range(world * SEGS_PER_PART)]
    mine = all_segs[rank * SEGS_PER_PART:(rank + 1) * SEGS_PER_PART]
    staged = [native.StagedSegment(s) for s in mine]
    group = native.SegmentGroup(staged)
    flags = native.PB_Q_COMBINE | native.PB_Q_ALL_RANKS
    for name, sql, exact in queries(all_segs):
        q = parse_sql(sql)
        cols = dictionary_columns(q, mine[0])
        agree_global_dictionaries(group, cols, [int(mine[0].columns[c].data_type) for c in cols], ex)
        exp, orc = expected(all_segs, q)
        for rep in range(2):                            # second pass: cached buffers, same answer
            res = native.execute(group, q, flags)
            check(f"rank {rank}: {name} (pass {rep})", res, exp, orc, q, exact, len(all_segs))   # EVERY rank holds the merged table
            assert res.comm_ms() > 0
            res.free()
    # a query whose group table is a hash table (raw LONG key); the filtered AVG keeps its own row count, which travels in
    # the tuples next to its sum
    d3 = all_segs[0].columns["c3"].dictionary_values()
    q = parse_sql(f"SET numGroupsLimit = 10000000; SELECT k0, SUM(m0), COUNT(*), AVG(m0) FILTER(WHERE c3 < {int(d3[len(d3) // 3])}) FROM t "
                  "GROUP BY k0 LIMIT 10000000")
    exp, orc = expected(all_segs, q)
    res = native.execute(group, q, flags)
    # hash tables are merged by a hash-partitioned all-to-all: every rank holds the groups whose key hashes to it (disjoint
    # partitions whose union is the merged table) and the statistics of the whole query
    t = res.tables[0]
    parts = ex.all_gather(t.rows())
    assert sum(len(p) for p in parts) == len(exp), (sum(len(p) for p in parts), len(exp))
    union = {}
    for p in parts:
        assert not (set(p) & set(union)), "partitions overlap"
        union.update(p)
    assert_rows_equal(union, exp, q, exact_float=True, what=f"rank {rank}: hash table (union of the partitions)")
    assert all(len(p) > 0 for p in parts), "a rank ended up without groups"
    st = t.stats
    assert st["num_docs_scanned"] == sum(o.stats["num_docs_scanned"] for o in orc) and st["num_segments"] == len(all_segs), st
    assert res.comm_ms() > 0
    res.free()
    ex.barrier()
    native.comm_destroy()
    print(f"MULTI_GPU_OK rank {rank}")


def run_devices(n_dev):
    native.init(list(range(n_dev)))
    all_segs = [segment(i) for i in range(n_dev * SEGS_PER_PART)]
    # interleave the segments over the devices: the group's segment order is not the device order
    staged = [native.StagedSegment(s, device_index=i % n_dev) for i, s in enumerate(all_segs)]
    group = native.SegmentGroup(staged)
    for name, sql, exact in queries(all_segs):
        q = parse_sql(sql)
        exp, orc = expected(all_segs, q)
        res = native.execute(group, q, native.PB_Q_COMBINE)
        check(f"{n_dev} devices: {name}", res, exp, orc, q, exact, len(all_segs))
        res.free()
        # per-segment tables come back in the caller's segment order whichever device ran them
        res = native.execute(group, q, 0)
        from tests.parity import oracle_rows
        assert len(res.tables) == len(all_segs)
        for i, (t, o) in enumerate(zip(res.tables, orc)):
            assert_rows_equal(t.rows(), oracle_rows(o), q, exact, what=f"{n_dev} devices: {name}: segment {i}")
            assert t.stats["num_docs_scanned"] == o.stats["num_docs_scanned"]
        res.free()
    print("MULTI_GPU_OK devices")


def run_single():
    """a communicator of ONE rank on one GPU: NCCL is loaded, ncclCommInitRank runs, PB_Q_ALL_RANKS is a no-op merge"""
    native.init(0)
    native.comm_init(1, 0, native.comm_unique_id())
    assert native.comm_info() == (True, 1, 0)
    all_segs = [segment(i) for i in range(3)]
    group = native.SegmentGroup([native.StagedSegment(s) for s in all_segs])
    for name, sql, exact in queries(all_segs):
        q = parse_sql(sql)
        exp, orc = expected(all_segs, q)
        res = native.execute(group, q, native.PB_Q_COMBINE | native.PB_Q_ALL_RANKS)
        check(f"single rank: {name}", res, exp, orc, q, exact, len(all_segs))
        res.free()
    native.comm_destroy()
    print("MULTI_GPU_OK single")


if __name__ == "__main__":
    if sys.argv[1] == "single":
        run_single()
    elif sys.argv[1] == "ranks":
        run_ranks(int(sys.argv[2]), int(sys.argv[3]), sys.argv[4])
    else:
        run_devices(int(sys.argv[2]))
