"""The fused candidate round of the specialised filter kernel (pb_filter_kernel<2, 4, W, K, RW>): a selective dense group-by
whose candidate leaves are row-group fields is aggregated inside the filter kernel, with no match list and no aggregation
kernel.  Every positive case asserts plan_info["fused_agg"] == 1, matches the exact reference, and matches a child process
that runs the same queries under PB_FUSED_AGG=0 (the filter kernel + pb_agg_rows_kernel) bit for bit: the inputs are INT
columns whose sums stay below 2^53, so every aggregate is exact on both paths.  Negative cases assert fused_agg == 0."""
import functools
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from pinot_b200 import datagen, native
from pinot_b200.query import parse_sql
from tests.reference import SegmentSource, assert_matches_reference, concat, evaluate_sql, reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLUMNS = datagen.CONFIG2_COLUMNS + ["c0", "c3", "x0"]
REPLAYS = 4                      # run 1 replays the cached plan, runs 2 and 3 its CUDA graph
CHILD_TIMEOUT_S = 900


@functools.lru_cache(maxsize=None)
def _tables():
    """name -> segments: config 2's shape; 20 segments of odd sizes (tail units, CTA ranges across segment ends); and
    dimension dictionaries drawn per segment (local -> global remaps that are not the identity)"""
    # (at least 10 000 docs each: c2 then has the same dictionary, and so the same width, in every segment)
    many = [10001, 10243, 12289, 16385, 20001, 11111, 13007, 10007, 15001, 10099, 18003, 10501, 14337, 10009, 12001, 10003, 17001,
            10021, 11003, 19999]
    return {"config2": datagen.make_table(8, 50_000, COLUMNS),
            "many": [datagen.make_segment_synth(i, n, COLUMNS) for i, n in enumerate(many)],
            "remap": datagen.make_table(4, 40_000, COLUMNS, vary_dim_dictionaries=True)}


def _where(segs, in_values=16):
    return datagen.config2_sql(segs, in_values).split(" WHERE ")[1].split(" GROUP BY ")[0]


def _queries():
    """case -> (table, SQL, expected fused_agg, expected row width or None)"""
    segs = _tables()["config2"]
    c1 = segs[0].columns["c1"].dictionary_values()
    c3 = segs[0].columns["c3"].dictionary_values()
    where = _where(segs)
    in_list = where.split(" AND ")[0]
    k2 = where.split(" AND ")[1]
    gb = " GROUP BY d0, d1, d2 LIMIT 100000"
    pre = "SET skipIndexes = 'c1=inverted,c3=inverted'; "                # scan c1 and c3 (both have inverted indexes)
    # 300 c2 values (3 %, less selective than c1's 1.6 %: c2 stays the candidate leaf) that no doc with c1 in the IN list
    # has: candidates exist, survivors do not
    src = concat([SegmentSource(s) for s in segs], ["c1", "c2"])
    sel_c1 = np.isin(src["c1"].values, [int(v) for v in in_list.split("(")[1].rstrip(")").split(", ")])
    absent = ", ".join(str(int(v)) for v in np.setdiff1d(np.unique(src["c2"].values), np.unique(src["c2"].values[sel_c1]))[:300])
    not_in = ", ".join(str(int(v)) for v in c1[15:])                     # NOT IN all but 15 of 1000 values: 1.5 % pass
    # per-segment dictionaries: 4 IN values from each segment's own c1 dictionary, so every segment streams a c1 set leaf
    remap = _tables()["remap"]
    remap_in = ", ".join(str(int(v)) for s in remap for v in s.columns["c1"].dictionary_values()[::250][:4])
    remap_sql = datagen.config2_sql(remap).replace(_where(remap).split(" AND ")[0], f"c1 IN ({remap_in})")
    return {
        "config2": ("config2", datagen.config2_sql(segs), 1, 4),
        "rw2": ("config2", f"{pre}SELECT d0, d1, d2, SUM(m0), COUNT(*) FROM t WHERE {where}{gb}", 1, 2),
        "rw8": ("config2", f"{pre}SELECT d0, d1, d2, SUM(m0), MIN(m1), MAX(m2), SUM(c0), COUNT(*) FROM t WHERE {where}{gb}", 1, 8),
        "two_cand": ("config2", f"{pre}SELECT d0, d1, d2, SUM(m0), MAX(m2) FROM t WHERE {where} AND c3 < {int(c3[len(c3) // 2])}{gb}", 1, None),
        "not_in": ("config2", f"{pre}SELECT d0, d1, d2, SUM(m0), MIN(m1), COUNT(*) FROM t WHERE c1 NOT IN ({not_in}) AND {k2}{gb}", 1, None),
        "no_survivors": ("config2", f"{pre}SELECT d0, d1, d2, SUM(m0), COUNT(*) FROM t WHERE {in_list} AND c2 IN ({absent}){gb}", 1, None),
        "many_segments": ("many", datagen.config2_sql(_tables()["many"]), 1, None),
        "remap": ("remap", remap_sql, 1, None),
        # not fused: 25 % pass (no candidate leaves), a raw candidate leaf
        "sel25": ("config2", datagen.config2_sql(segs, 500), 0, None),
        "raw_leaf": ("config2", f"{pre}SELECT d0, d1, d2, SUM(m0), COUNT(*) FROM t WHERE {in_list} AND x0 < 0.5{gb}", 0, None),
    }


def _run(names):
    """case -> [(rows, plan_info, num_docs_scanned) per run]; config2 runs REPLAYS times (plan cache, CUDA graph)"""
    native.init()
    qs = _queries()
    out = {}
    groups = {}
    try:
        for name in names:
            table, sql, _, _ = qs[name]
            if table not in groups:
                staged = [native.StagedSegment(s) for s in _tables()[table]]
                groups[table] = (staged, native.SegmentGroup(staged))
            g = groups[table][1]
            q = parse_sql(sql)
            # the first call of a query stages its columns and builds its row groups: its kernels run in waves behind
            # those copies, a plan that is neither cached nor fused
            native.execute(g, q, native.PB_Q_COMBINE).free()
            runs = []
            for _ in range(REPLAYS if name == "config2" else 1):
                res = native.execute(g, q, native.PB_Q_COMBINE)
                t = res.tables[0]
                runs.append((t.rows(), res.plan_info, t.stats["num_docs_scanned"]))
                res.free()
            out[name] = runs
    finally:
        for staged, g in groups.values():
            g.release()
            for s in staged:
                s.release()
    return out


def _child(env_extra, names, tmp_path):
    path = str(tmp_path / ("child_" + "_".join(f"{k}={v}" for k, v in env_extra.items()) + ".pkl"))
    env = {k: v for k, v in os.environ.items() if k not in ("PB_FUSED_AGG", "PB_AGG_SMEM_MIN")}
    env.update(env_extra)
    env["PYTHONDONTWRITEBYTECODE"] = "1"
    p = subprocess.run([sys.executable, "-m", "tests.test_gpu_fused_agg", path, *names], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=CHILD_TIMEOUT_S)
    assert p.returncode == 0, (p.stdout + p.stderr)[-6000:]
    with open(path, "rb") as f:
        return pickle.load(f)


# (in this order: a query whose columns all lie in an existing row group reads that group, so the 2-word group must be
# built before config 2's 4-word one)
POSITIVE = ["rw2", "config2", "rw8", "two_cand", "not_in", "no_survivors", "many_segments", "remap"]
NEGATIVE = ["sel25", "raw_leaf"]


@pytest.fixture(scope="module")
def fused_runs():
    return _run(POSITIVE + NEGATIVE)


@pytest.mark.gpu
@pytest.mark.parametrize("name", POSITIVE + NEGATIVE)
def test_fused_against_reference(name, fused_runs):
    table, sql, fused, rw = _queries()[name]
    q = parse_sql(sql)
    src = concat([SegmentSource(s) for s in _tables()[table]])
    ref = reference(src, q)
    n_match = int(evaluate_sql(src, q.filter).sum())
    if name == "no_survivors":
        assert n_match == 0 and not ref
    for rows, pi, scanned in fused_runs[name]:
        assert pi["fused_agg"] == fused, f"{name}: {pi}"
        if fused:
            # reported as the rows-kernel path it replaces, without a CTA table
            assert pi["agg_kernel"] == 3 and pi["filter_kernel"] == 3 and pi["st_replicas"] == 0 and pi["exact_int_mask"] == 0, f"{name}: {pi}"
            if rw:
                assert pi["rows_rw"] == rw, f"{name}: {pi}"
        assert_matches_reference(rows, ref, q, f"{name}: {sql}")
        assert scanned == n_match, (name, scanned, n_match)
    first = fused_runs[name][0][0]
    for rows, _, _ in fused_runs[name][1:]:
        assert rows == first, f"{name}: a plan-cache / graph replay differs from the first run"


@pytest.mark.gpu
def test_fused_matches_the_two_kernel_path(fused_runs, tmp_path):
    """PB_FUSED_AGG=0 in a child: the same queries through the filter kernel's match list and pb_agg_rows_kernel give the
    same tables bit for bit"""
    unfused = _child({"PB_FUSED_AGG": "0"}, POSITIVE, tmp_path)
    for name in POSITIVE:
        rows, pi, scanned = unfused[name][0]
        assert pi["fused_agg"] == 0 and pi["agg_kernel"] == 3, (name, pi)
        assert rows == fused_runs[name][0][0], f"{name}: fused and two-kernel results differ"
        assert scanned == fused_runs[name][0][2], name


@pytest.mark.gpu
def test_no_fusion_when_the_cta_table_is_forced(fused_runs, tmp_path):
    """PB_AGG_SMEM_MIN=0: the rows kernel would take its CTA-private table, so the call keeps the two kernels"""
    forced = _child({"PB_AGG_SMEM_MIN": "0"}, ["config2"], tmp_path)
    rows, pi, _ = forced["config2"][0]
    assert pi["fused_agg"] == 0 and pi["st_replicas"] > 0, pi
    assert rows == fused_runs["config2"][0][0]


if __name__ == "__main__":
    # child mode: python -m tests.test_gpu_fused_agg OUT.pkl CASE...
    result = _run(sys.argv[2:])
    with open(sys.argv[1], "wb") as f:
        pickle.dump(result, f)
