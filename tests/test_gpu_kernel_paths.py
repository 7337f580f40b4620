"""The tuning knobs of libpinot_b200.so (DESIGN.md §9) each switch a kernel path off or force one on.  The library reads
every knob once per process, so each setting runs the device fuzz (a fixed, smaller seed set) and the deterministic
cases of tests/test_gpu_fuzz.py in a child pytest process with only that variable changed.  A final test
checks from the children's plan logs that the default knobs and PB_AGG_SMEM_MIN=0 together reached every kernel path."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = "1,2"                    # seed 1: more than 16 segments, LONG sums past the exact bound; seed 2: 2^24 + 1 slots
MAX_DOCS = "150000"
CHILD_TIMEOUT_S = 600
SETTINGS = [
    {}, {"PB_AGG_SMEM_MIN": "0"}, {"PB_AGG_SMEM": "0"}, {"PB_AGG_ROWS": "0"}, {"PB_ROW_GROUPS": "0"},
    {"PB_AGG_EXACT_INT": "0"}, {"PB_FILTER_SPEC": "0"}, {"PB_UNIT": "1"}, {"PB_GATHER_LEAF_PERMILLE": "0"},
    {"PB_GATHER_LEAF_PERMILLE": "1000"}, {"PB_SPARSE_MAX": "0"}, {"PB_SPARSE_MAX": "1024"}, {"PB_PLAN_CACHE": "0"}, {"PB_GRAPH": "0"},
]
KNOBS = {k for s in SETTINGS for k in s}
_runs = {}


def _name(setting):
    return ",".join(f"{k}={v}" for k, v in setting.items()) or "defaults"


def run_child(setting, tmp_dir):
    """run the fuzz module under one setting (memoised per session); returns (returncode, output tail, plan log records)"""
    name = _name(setting)
    if name not in _runs:
        log = os.path.join(tmp_dir, name.replace("=", "_").replace(",", "__") + ".jsonl")
        env = {k: v for k, v in os.environ.items() if k not in KNOBS}
        env.update(setting)
        env.update({"PB_FUZZ_SEEDS": SEEDS, "PB_FUZZ_MAX_DOCS": MAX_DOCS, "PB_FUZZ_PLAN_LOG": log, "PYTHONDONTWRITEBYTECODE": "1"})
        cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider",
               os.path.join(ROOT, "tests", "test_gpu_fuzz.py")]
        try:
            p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=CHILD_TIMEOUT_S)   # kills the child on timeout
            rc, out = p.returncode, (p.stdout + p.stderr)[-6000:]
        except subprocess.TimeoutExpired as e:
            rc, out = -1, f"timed out after {CHILD_TIMEOUT_S} s\n" + str(e.stdout or "")[-4000:]
        recs = []
        if os.path.exists(log):
            with open(log) as f:
                recs = [json.loads(line) for line in f if line.strip()]
        _runs[name] = (rc, out, recs)
    return _runs[name]


@pytest.fixture(scope="module")
def tmp_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kernel_paths"))


@pytest.mark.gpu
@pytest.mark.parametrize("setting", SETTINGS, ids=_name)
def test_fuzz_under_knob(setting, tmp_dir):
    """Every fuzz query and every deterministic case pass under the setting: an error from the library (PB_ERR_UNSUPPORTED
    included) fails the child, so a knob may not decline what the defaults run."""
    rc, out, recs = run_child(setting, tmp_dir)
    assert rc == 0, f"{_name(setting)}:\n{out}"
    assert recs, f"{_name(setting)}: no plan was logged"


def _reached(recs):
    got = {}
    for r in recs:
        got.setdefault("agg_kernel", set()).add(r["agg_kernel"])
        if r["agg_kernel"] == 3:
            got.setdefault("rows_rw", set()).add(r["rows_rw"])
            got.setdefault("exact", set()).add(r["exact_int_mask"] != 0)
        got.setdefault("table", set()).add((r["table_mode"], r["key_words"]) if r["table_mode"] == 2 else (r["table_mode"], 0))
        got.setdefault("filter", set()).add(r["filter_kernel"])
        got.setdefault("cand_leaf", set()).add(r["cand_leaf"])
        got.setdefault("st_replicas", set()).add(r["st_replicas"])
        got.setdefault("many_segs_rows", set()).add(r["n_segs"] > 16 and r["agg_kernel"] == 3)
    return got


@pytest.mark.gpu
def test_every_kernel_path_is_reached(tmp_dir):
    """Under the default knobs and PB_AGG_SMEM_MIN=0 together: every aggregation kernel, every row width, exact-integer
    mode on and off, keyless / dense / hash-64 / hash-128 tables, the general filter kernel at U=1 and U=2, the specialised
    one, candidate leaves, pb_agg_rows_kernel over more than 16 segments, and CTA tables of 1 (at the shared-memory budget)
    and 32 replicas"""
    recs = []
    for s in ({}, {"PB_AGG_SMEM_MIN": "0"}):
        rc, out, r = run_child(s, tmp_dir)
        assert rc == 0, f"{_name(s)}:\n{out}"
        recs += r
    got = _reached(recs)
    want = {"agg_kernel": {1: "pb_agg_kernel", 2: "pb_agg_smem_kernel", 3: "pb_agg_rows_kernel"},
            "rows_rw": {2: "RW=2", 4: "RW=4", 8: "RW=8"}, "exact": {True: "exact-integer sums", False: "double sums in the rows kernel"},
            "table": {(0, 0): "keyless", (1, 0): "dense", (2, 1): "hash, 1 key word", (2, 2): "hash, 2 key words"},
            "filter": {1: "general filter U=1", 2: "general filter U=2", 3: "specialised filter"},
            "cand_leaf": {1: "candidate leaves"}, "many_segs_rows": {True: "pb_agg_rows_kernel over > 16 segments"},
            "st_replicas": {1: "one CTA table at the 200 KB budget", 32: "32 CTA table replicas"}}
    missing = [label for k, opts in want.items() for v, label in opts.items() if v not in got.get(k, set())]
    assert not missing, f"kernel paths no fuzz call reached: {missing}"
