"""Differential tests of the host side of the SQL surface against the LIVE reference extension (oracle/_ref/cpu/vector.so), each
in its own process: the vector_as_* encoders on drawn JSON / BLOB inputs (number formats, separators, brackets, dimension
arguments) and vector_quantize builds on drawn tables (5 source types, dims 1..40, NULL rows, NaN / Inf / huge values, constant
and non-negative columns, both qtypes, several max_memory settings) — rows, error strings, shadow-table bytes and metadata
must be identical.  CPU only (without a GPU vector_quantize runs its host loops; the GPU loops are pinned to the same bytes by
test_gpu_parity.py / test_sql_surface.py / test_gpu_quantizer.py, which also runs the quantize scripts below on the GPU).  Seeds are fixed; 24 000 encoder statements and 240 table scripts were run once
offline without a mismatch."""
import os
import random

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import refreplay
from tests.sqlrun import OURS, REF_CPU, blob, run_sql

needs_ref = pytest.mark.skipif(not os.path.exists(REF_CPU + ".so") and not refreplay.available("sql"),
                               reason="oracle/_ref not built and no recorded reference outputs")

NUMS = ["0", "1", "-1", "2.5", "-3e2", "1e-7", "+5", ".5", "5.", "1e400", "-1e400", "1e-400", "nan", "NaN", "inf", "-inf", "Infinity", "0x10", "1_000", "",
        "--1", "1e", "1e+", "127", "-128", "128", "-129", "255", "256", "3.9", "-3.9", "65504", "65520", "70000", "1e38", "3.5e38", "0.1", "1e-45", "007", "1.0.0",
        "1,5", "true", "null", "\"1\"", "1f", "1d", " 1 ", "1 2", "\t3", "4\n"]
FUNCS = ["vector_as_f32", "vector_as_f16", "vector_as_bf16", "vector_as_i8", "vector_as_u8"]


def _json_text(rng):
    n = rng.choice([0, 1, 2, 3, 4, 5, 8])
    toks = [rng.choice(NUMS) if rng.random() < 0.35 else repr(round(rng.uniform(-300, 300), rng.choice([0, 1, 3]))) for _ in range(n)]
    sep = rng.choice([",", ", ", " , ", ",  ", ",\n"])
    body = sep.join(toks)
    if rng.random() < 0.1:
        body += ","
    if rng.random() < 0.05:
        body = "," + body
    if rng.random() < 0.05:
        body = body.replace(sep, sep + sep, 1)
    form = rng.random()
    if form < 0.75:
        return "[" + body + "]"
    if form < 0.8:
        return body
    if form < 0.85:
        return "[" + body
    if form < 0.9:
        return body + "]"
    if form < 0.93:
        return "[[" + body + "]]"
    if form < 0.96:
        return "[" + body + "] x"
    return "  [ " + body + " ]  "


def _encoder_stmt(rng):
    f = rng.choice(FUNCS)
    r = rng.random()
    if r < 0.7:
        arg = "'" + _json_text(rng).replace("'", "''") + "'"
    elif r < 0.95:
        arg = "x'" + bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 2, 3, 4, 6, 8, 12, 16, 5, 7]))).hex() + "'"
    else:
        arg = rng.choice(["42", "NULL", "4.5", "''", "'[]'"])
    if rng.random() < 0.6:
        return f"SELECT hex({f}({arg}))"
    return f"SELECT hex({f}({arg}, {rng.choice(['0', '1', '2', '3', '4', '5', '8', '-1', 'NULL', chr(39) + '3' + chr(39), '2.0', '1000000'])}))"


@needs_ref
@pytest.mark.parametrize("seed", [3, 17])
def test_encoders_match_live_reference(seed):
    rng = random.Random(seed)
    script = [_encoder_stmt(rng) for _ in range(400)]
    ours, ref = run_sql(OURS, script), run_sql(REF_CPU, script)
    for s, a, b in zip(script, ours, ref):
        assert a == b, (s, a, b)


TYPES = [(po.F32, "FLOAT32"), (po.F16, "FLOAT16"), (po.BF16, "FLOATB16"), (po.I8, "INT8"), (po.U8, "UINT8")]
SPECIALS = [np.nan, np.inf, -np.inf, 3.0e38, -3.0e38, 65504.0, 1e-30, 0.0, -0.0]


def _quantize_script(seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    s = []
    for t in range(3):
        vt, tname = TYPES[rng.integers(5)]
        dim, n = int(rng.integers(1, 41)), int(rng.choice([0, 1, 2, 7, 30, 120]))
        tb = f"q{t}"
        s += [f"CREATE TABLE {tb} (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('{tb}', 'e', 'type={tname},dimension={dim}')"]
        x = (rng.standard_normal((max(n, 1), dim)) * float(rng.choice([1e-3, 1.0, 40.0, 1e4]))).astype(np.float32)
        if vt in (po.I8, po.U8):
            x = np.clip(np.round(x), -128 if vt == po.I8 else 0, 127 if vt == po.I8 else 255)
        if vt in (po.F32, po.F16, po.BF16) and rng.random() < 0.4:
            for _ in range(int(rng.integers(1, 4))):
                x[rng.integers(x.shape[0]), rng.integers(dim)] = rng.choice(SPECIALS)
        if rng.random() < 0.2:
            x[:] = x[0, 0]                      # constant column: max == min
        if rng.random() < 0.15:
            x = np.abs(x)                       # no negative value: the UINT8 default
        with np.errstate(over="ignore"):
            xx = po.convert(x, vt)
        ids = rng.permutation(1000)[:n] - 300
        for i in range(n):
            if rng.random() < 0.05:
                s.append([f"INSERT INTO {tb}(id, e) VALUES (?, NULL)", [int(ids[i])]])
            else:
                s.append([f"INSERT INTO {tb}(id, e) VALUES (?, ?)", [int(ids[i]), blob(xx[i])]])
        for _ in range(2):
            opt = rng.choice(["", "qtype=UINT8", "qtype=INT8", "max_memory=1KB", "qtype=INT8,max_memory=2KB", "max_memory=0", "qtype=UINT8,max_memory=512"])
            s.append(f"SELECT vector_quantize('{tb}', 'e'" + (f", '{opt}'" if opt else "") + ")")
            s.append(f"SELECT rowid1, rowid2, counter, hex(data) FROM vector0_{tb}_e")
            s.append(f"SELECT key, value FROM _sqliteai_vector WHERE tblname='{tb}' ORDER BY key")
            s.append(f"SELECT vector_quantize_memory('{tb}', 'e')")
    return s


@needs_ref
@pytest.mark.parametrize("seed", [1, 2, 5, 8, 13, 21])
def test_quantize_builds_match_live_reference(seed):
    script = _quantize_script(seed)
    ours, ref = run_sql(OURS, script, env={"CUDA_VISIBLE_DEVICES": ""}), run_sql(REF_CPU, script)
    for s, a, b in zip(script, ours, ref):
        assert a == b, (s if isinstance(s, str) else s[0], str(a)[:300], str(b)[:300])


OPT_KEYS = ["type", "dimension", "distance", "normalized", "qtype", "max_memory", "bogus", "TYPE", "Dimension", " type", "dim", ""]
OPT_VALS = {"type": ["FLOAT32", "float32", "FLOAT16", "FLOATB16", "BFLOAT16", "INT8", "UINT8", "F32", "FLOAT64", "", "int8 ", " INT8"],
            "dimension": ["4", "8", "0", "-3", "1e2", "4.5", "abc", "", "3 ", "0x10", "+7"],
            "distance": ["L2", "l2", "SQUARED_L2", "COSINE", "cosine", "DOT", "INNER", "L1", "MANHATTAN", "", "EUCLIDEAN"],
            "normalized": ["0", "1", "true", "yes", ""],
            "qtype": ["UINT8", "INT8", "int8", "1BIT", "", "AUTO"],
            "max_memory": ["0", "1KB", "1kb", "2MB", "1GB", "512", "-1", "abc", "1.5MB", "10 KB", ""]}


def _option_string(rng):
    parts = []
    for _ in range(rng.choice([0, 1, 2, 3, 4, 5])):
        k = rng.choice(OPT_KEYS)
        v = rng.choice(OPT_VALS.get(k.strip().lower(), ["1", "x", ""]))
        eq = rng.choice(["=", " = ", "= ", " =", "==", ":", ""]) if rng.random() < 0.25 else "="
        parts.append(f"{k}{eq}{v}")
    s = (rng.choice([",", ", ", " ,", ",,", ";"]) if rng.random() < 0.3 else ",").join(parts)
    if rng.random() < 0.1:
        s = "," + s
    if rng.random() < 0.1:
        s += ","
    return s


@needs_ref
@pytest.mark.parametrize("block", [0, 1])
def test_option_strings_match_live_reference(block):
    """vector_init / vector_quantize option strings (the key=value parser, unknown keys, bad values): same rows, same error
    strings, same metadata.  One connection per table, because the reference returns from a vector_quantize with an invalid
    option string with its transaction open and the emptied shadow table in place (deviation 9: ours rolls both back) — the
    one statement after such a failure that is not compared.  Dimensions beyond 2^29 are left out: there the reference fails in
    sqlite3_malloc64(dim * 4) with an empty error message before it looks at a row, ours reports the row's blob as too short."""
    for seed in range(40 * block, 40 * block + 40):
        rng = random.Random(1000 + seed)
        opts = _option_string(rng)
        if rng.random() < 0.5:
            opts = "type=FLOAT32,dimension=4," + opts
        script = ["CREATE TABLE o (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('o', 'e', '{opts}')",
                  "SELECT key, value FROM _sqliteai_vector WHERE tblname='o' ORDER BY key",
                  ["INSERT INTO o(id, e) VALUES (1, ?)", [{"hex": "0000803f000000400000404000008040"}]],
                  ["INSERT INTO o(id, e) VALUES (2, ?)", [{"hex": "000080bf0000004000004040000080c0"}]],
                  f"SELECT vector_quantize('o', 'e', '{_option_string(rng)}')",
                  "SELECT key, value FROM _sqliteai_vector WHERE tblname='o' ORDER BY key",
                  "SELECT count(*), sum(length(data)) FROM vector0_o_e"]
        ours, ref = run_sql(OURS, script, env={"CUDA_VISIBLE_DEVICES": ""}), run_sql(REF_CPU, script)
        quantize_failed = ours[5] == ref[5] and ("error" in ours[5] or ours[5]["rows"] == [[None]])     # error, or the silent NULL of a rejected option string
        for i, (s, a, b) in enumerate(zip(script, ours, ref)):
            if i == 7 and quantize_failed:
                continue
            assert a == b, (seed, script[1], script[5], s if isinstance(s, str) else s[0], a, b)


ARG_VALUES = ["NULL", "1", "-1", "0", "2.5", "'t'", "'e'", "'nope'", "''", "x''", "x'0000803f00000040'", "'[1,2]'", "'type=FLOAT32,dimension=2'", "'qtype=INT8'",
              "20", "'20'", "1e10", "9223372036854775807"]
ARG_SCALARS = [("vector_version", [0]), ("vector_backend", [0]), ("vector_init", [3]), ("vector_quantize", [2, 3]), ("vector_quantize_memory", [2]),
               ("vector_quantize_preload", [2]), ("vector_quantize_cleanup", [2])]
ARG_TVFS = [("vector_full_scan", 4), ("vector_quantize_scan", 4), ("vector_full_scan_stream", 3), ("vector_quantize_scan_stream", 3),
            ("vector_full_scan_batch", 4), ("vector_quantize_scan_batch", 4),
            ("vector_full_scan_filtered", 5), ("vector_quantize_scan_filtered", 5),
            ("vector_full_scan_batch_filtered", 5), ("vector_quantize_scan_batch_filtered", 5),
            ("vector_full_scan_batch_sets", 6), ("vector_quantize_scan_batch_sets", 6),
            ("vector_full_scan_grouped", 6), ("vector_quantize_scan_grouped", 6),
            ("vector_full_scan_range", 4), ("vector_quantize_scan_range", 4),
            ("vector_full_scan_range_filtered", 5), ("vector_quantize_scan_range_filtered", 5),
            ("vector_quantize_scan_rerank", 5), ("vector_quantize_scan_rerank_batch", 5)]


def _arg_stmt(rng):
    if rng.random() < 0.5:
        f, ar = rng.choice(ARG_SCALARS)
        n = rng.choice(ar) if rng.random() < 0.85 else rng.choice([0, 1, 2, 3, 4])
        args = [rng.choice(ARG_VALUES) for _ in range(n)]
        if n >= 2 and rng.random() < 0.6:
            args[0], args[1] = "'t'", rng.choice(["'e'", "'e'", "'zz'"])
        return f"SELECT {f}({', '.join(args)})"
    f, n = rng.choice(ARG_TVFS)
    n = n if rng.random() < 0.85 else rng.choice([1, 2, 3, 4, 5])
    args = [rng.choice(ARG_VALUES) for _ in range(n)]
    if n >= 2 and rng.random() < 0.7:
        args[0], args[1] = "'t'", rng.choice(["'e'", "'e'", "'zz'"])
    return f"SELECT * FROM {f}({', '.join(args)}) LIMIT 3"


def test_random_argument_types_never_crash():
    """every SQL function and table-valued module with drawn argument counts and types (NULL, integers, reals, text, blobs, huge
    values): each statement ends in rows or an error, the process survives.  (No comparison here: the unmodified reference
    segfaults on most of these scripts — NULL / non-text names, missing arguments — so only our side is driven.)"""
    for seed in range(60):
        rng = random.Random(seed)
        script = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)"]
        if rng.random() < 0.7:
            script.append("SELECT vector_init('t', 'e', 'type=FLOAT32,dimension=2')")
        script += [_arg_stmt(rng) for _ in range(8)]
        out = run_sql(OURS, script, env={"CUDA_VISIBLE_DEVICES": ""})
        assert len(out) == len(script) and all(("rows" in o) != ("error" in o) for o in out), (seed, script)
