"""The table-valued functions check a call in one order: the argument count, then each argument on its own in position order
(SQL type, BLOB size, the range of k, limit and candidates), then the context, the query against the column, query_sets
against the queries, the quantization table and staging.  So a negative k, a negative limit or candidates out of range is
reported before anything that needs the column, on every module that takes one.  The SQL runs with no CUDA device visible, so
staging always fails (the column also holds a short vector blob, which fails it on a device too), and the column is never
quantized."""
import pytest

from tests.sqlrun import OURS, run_sql

SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", "SELECT vector_init('t','e','type=FLOAT32,dimension=2')",
         "INSERT INTO t(id, e) VALUES (1, x'0000803f00000040'), (2, x'01')"]
Q = "x'0000803f00000040'"
PAIRS = "x'03000000000000000100000000000000'"
ROWIDS = "x'0100000000000000'"

# every module with a k: the arguments after k
K_MODULES = {f"vector_{kind}_scan{suffix}": tail
             for kind in ("full", "quantize")
             for suffix, tail in (("", ""), ("_batch", ""), ("_filtered", f",{ROWIDS}"), ("_batch_filtered", f",{ROWIDS}"),
                                  ("_batch_sets", f",{PAIRS},NULL"), ("_grouped", f",{PAIRS},NULL"))}
K_MODULES.update({"vector_quantize_scan_rerank": ",10", "vector_quantize_scan_rerank_batch": ",10"})


def _errors(stmts):
    out = run_sql(OURS, SETUP + stmts, env={"CUDA_VISIBLE_DEVICES": ""})[len(SETUP):]
    return [o.get("error") for o in out]


def test_every_k_module_reports_negative_k_before_the_column():
    assert len(K_MODULES) == 14
    names = sorted(K_MODULES)
    stmts = []
    for fn in names:
        tail = K_MODULES[fn]
        stmts += [f"SELECT * FROM {fn}('t','e',{Q},-1{tail})",          # the column can be neither staged nor found quantized
                  f"SELECT * FROM {fn}('nope','e',{Q},-1{tail})",       # before the context
                  f"SELECT * FROM {fn}('t','e',x'0102',-1{tail})"]      # before the query's length
    errs = _errors(stmts)
    for i, fn in enumerate(names):
        assert errs[3 * i: 3 * i + 3] == [f"{fn}: k must not be negative."] * 3, (fn, errs[3 * i: 3 * i + 3])


def test_the_column_errors_stand_without_a_negative_k():
    """the same calls with k = 3: the staging or quantization-table error each module reports"""
    names = sorted(K_MODULES)
    errs = _errors([f"SELECT * FROM {fn}('t','e',{Q},3{K_MODULES[fn]})" for fn in names])
    for fn, e in zip(names, errs):
        if "_quantize_" in fn:
            assert e.startswith("Quantization table not found for table 't' and column 'e'."), (fn, e)
        else:
            assert e.startswith("Invalid vector blob found at rowid 2.") or e.startswith("vector_full_scan: "), (fn, e)


@pytest.mark.parametrize("fn", ["vector_full_scan_grouped", "vector_quantize_scan_grouped"])
def test_grouped_negative_k_and_limit_reports_k(fn):
    assert _errors([f"SELECT * FROM {fn}('t','e',{Q},-1,{PAIRS},-1)", f"SELECT * FROM {fn}('t','e',{Q},3,{PAIRS},-1)"]) == [
        f"{fn}: k must not be negative.", f"{fn}: limit must not be negative."]


@pytest.mark.parametrize("fn", ["vector_quantize_scan_rerank", "vector_quantize_scan_rerank_batch"])
def test_rerank_candidates_out_of_range_before_the_quantization_table(fn):
    msg = f"{fn}: candidates must be between 0 and 2147483647."
    assert _errors([f"SELECT * FROM {fn}('t','e',{Q},3,-1)", f"SELECT * FROM {fn}('t','e',{Q},3,2147483648)",
                    f"SELECT * FROM {fn}('nope','e',{Q},3,-1)"]) == [msg] * 3
