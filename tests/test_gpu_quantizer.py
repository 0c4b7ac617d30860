"""The GPU side of vector_quantize on its own: quant_minmax_kernel and quant_encode_kernel (csrc/quant_kernels.cuh) driven through
vsb_quantizer_* (csrc/quantize.inc).  The shadow-table chunks they write are what vector_quantize_scan loads later, so every
output byte must equal the reference's.  -m gpu.

Every encoded buffer is compared with two references, exactly (the output is bytes, no tolerance applies):
  (a) oracle.build_quant_buffer / oracle.quant_params, pinned to the reference by test_oracle_vs_reference.py;
  (b) `restate_bytes` below, a numpy statement of the reference rule (sqlite-vector.c:495-757, :1295-1311), asserted equal to (a)
      on every input so that neither can drift.

(1) rowid bytes at every small dimension, including dims below 8 where a row has fewer element threads than rowid bytes;
(2) every f16 / bf16 bit pattern and every int8 / uint8 value, both qtypes, several (offset, scale) pairs;
(3) f32 rounding and range edges: exact halves, their neighbours, values past +-2^31 (x86 cvttss2si), +-Inf, NaN, and inputs on
    which a fused multiply-add would round differently;
(4) the min / max pass against the reference's sequential loop, fed in blocks around the staging size;
(5) non-finite scales (constant, all-zero and all-NaN columns);
(6) the staging loop over several blocks, retained / streamed / overflowed retention, and retained sub-range encodes;
(7) vector_quantize through SQL on the GPU: the recorded fuzz scripts, and tables of dims 1..7 with extreme rowids."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests.sqlrun import OURS, REF_CPU, blob, run_sql
from tests.test_sql_fuzz import _quantize_script, needs_ref

pytestmark = pytest.mark.gpu

TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
TYPE_SQL = {po.F32: "FLOAT32", po.F16: "FLOAT16", po.BF16: "FLOATB16", po.U8: "UINT8", po.I8: "INT8"}
INT_MIN = -(2 ** 31)
INT64_MIN, INT64_MAX = -(2 ** 63), 2 ** 63 - 1
FLT_MAX = float(np.finfo(np.float32).max)
STAGE_BYTES = 16 << 20                                  # kQuantStage: bytes per pinned staging buffer


def _quantizer(vtype, dim, retain_rows=0):
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    assert eng.device_count() >= 1, "no CUDA device: the GPU tests must not pass on a fallback"
    return vs.api.Quantizer(vtype, dim, retain_rows=retain_rows, engine=eng)


def stage_rows(vtype, dim):
    return max(1, STAGE_BYTES // (dim * po.ELEM_SIZE[vtype]))


def as_f32(vtype, x):
    """elements as fp32, like the reference's per-type loops"""
    if vtype == po.F32:
        return np.array(x, dtype=np.float32)
    if vtype == po.F16:
        return x.view(np.float16).astype(np.float32)
    if vtype == po.BF16:
        return (x.astype(np.uint32) << np.uint32(16)).view(np.float32)
    return x.astype(np.float32)


def scaled(vtype, x, offset, scale):
    """s = (v - offset) * scale, two separately rounded fp32 operations"""
    with np.errstate(all="ignore"):
        return (as_f32(vtype, x) - np.float32(offset)) * np.float32(scale)


def q_from_s(vtype, s, qtype):
    """round half away from zero; f32 sources: x86 (int) cast (NaN or |r| >= 2^31 -> INT_MIN), then clamp; other sources:
    q_round_u8 / q_round_s8 (sqlite-vector.c:495-515).  Returns int64 values in [-128, 255]."""
    with np.errstate(all="ignore"):
        r = s + np.where(s < 0, np.float32(-0.5), np.float32(0.5))
        t = np.trunc(np.where(np.isfinite(r), r, np.float32(0))).astype(np.int64)
        if vtype == po.F32:
            i = np.where(np.isnan(r) | ~(np.abs(r) < np.float32(2.0 ** 31)), INT_MIN, t)
            return np.clip(i, 0, 255) if qtype == po.Q_U8 else np.clip(i, -128, 127)
        fin = np.isfinite(s)
        if qtype == po.Q_U8:
            inner = np.where(r >= 255, 255, np.where(r <= 0, 0, t))
            return np.where(fin, inner, np.where(s > 0, 255, 0))
        inner = np.where(r >= 127, 127, np.where(r <= -128, -128, t))
        return np.where(fin, inner, np.where(s > 0, 127, np.where(s < 0, -128, 0)))


def restate_bytes(vtype, x, rowids, offset, scale, qtype):
    n, dim = x.shape
    out = np.empty((n, 8 + dim), dtype=np.uint8)
    out[:, :8] = np.ascontiguousarray(rowids, dtype="<i8").view(np.uint8).reshape(n, 8)
    out[:, 8:] = (q_from_s(vtype, scaled(vtype, x, offset, scale), qtype) & 0xFF).astype(np.uint8)
    return out.reshape(-1)


def expected(oracle, vtype, x, rowids, offset, scale, qtype):
    want = oracle.build_quant_buffer(vtype, x, rowids, offset, scale, qtype)
    mine = restate_bytes(vtype, x, rowids, offset, scale, qtype)
    assert np.array_equal(want, mine), ("the numpy restatement disagrees with the oracle", _diff(mine, want, x.shape[1]))
    return want


def _diff(got, want, dim):
    """first mismatching (row, byte, got, want); bytes 0..7 of a row are its rowid"""
    bad = np.nonzero(got != want)[0]
    return [(int(i // (8 + dim)), int(i % (8 + dim)), int(got[i]), int(want[i])) for i in bad[:8]], int(bad.size)


def check_bytes(got, want, dim, *ctx):
    assert got.shape == want.shape, ctx
    assert np.array_equal(got, want), (*ctx, "(row, byte, got, want), mismatches:", _diff(got, want, dim))


def ref_minmax(vtype, x):
    """the reference's loop (sqlite-vector.c:1202-1256): lo = FLT_MAX, hi = -FLT_MAX, `val < lo`, `val > hi`, `val < 0`"""
    v = as_f32(vtype, x).ravel()
    ok = v[~np.isnan(v)]
    lo, hi = np.float32(FLT_MAX), np.float32(-FLT_MAX)
    if ok.size:
        lo, hi = min(lo, ok.min()), max(hi, ok.max())
    return float(lo), float(hi), bool((v < 0).any())


def params(lo, hi, qtype):
    """scale / offset from the min / max pass, in fp32 like vector_ext.c (:1265-1268)"""
    lo, hi = np.float32(lo), np.float32(hi)
    with np.errstate(all="ignore"):
        if qtype == po.Q_U8:
            return float(np.float32(255.0) / (hi - lo)), float(lo)
        return float(np.float32(127.0) / max(abs(lo), abs(hi))), 0.0


def same_value(a, b):
    return a == b or (np.isnan(a) and np.isnan(b))


def check_minmax(oracle, qz, vtype, x, *ctx):
    """minmax_result() equals the reference loop (+-0 compared by value), and the parameters derived from it equal the oracle's
    for AUTO and both forced qtypes; returns (lo, hi, negative)"""
    lo, hi, neg = qz.minmax_result()
    wlo, whi, wneg = ref_minmax(vtype, x)
    assert (lo, hi, neg) == (wlo, whi, wneg), (*ctx, (lo, hi, neg), (wlo, whi, wneg))
    for qin in (po.Q_AUTO, po.Q_U8, po.Q_S8):
        osc, ooff, oqt = oracle.quant_params(vtype, x, qin)
        qt = qin if qin != po.Q_AUTO else (po.Q_S8 if neg else po.Q_U8)
        sc, off = params(lo, hi, qt)
        assert qt == oqt and same_value(sc, osc) and same_value(off, ooff), (*ctx, qin, (sc, off, qt), (osc, ooff, oqt))
    return lo, hi, neg


# ------------------------------------------------------------------------------------------------ (1) rowid bytes
ROWIDS = [INT64_MIN, INT64_MAX, -1, 0, 255, 256, 2 ** 32, 2 ** 56 - 1]


@pytest.mark.parametrize("dim", list(range(1, 18)) + [31, 32, 33])
@pytest.mark.parametrize("vtype", TYPES)
def test_rowid_bytes_every_small_dim(oracle, vtype, dim):
    """all 8 rowid bytes of every row, at dims below, at and above 8.  One quantizer first encodes a block whose rowids are all
    -1 and then a block of small and extreme rowids into the same output buffer, so a byte the kernel fails to write keeps 0xFF
    whatever the allocator handed out."""
    rng = np.random.Generator(np.random.PCG64(1000 * vtype + dim))
    rowids = np.array(ROWIDS + [int(v) for v in rng.integers(INT64_MIN, 0, 24)] + [1, 2, 3, 5], dtype=np.int64)
    n = rowids.size
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32) * 3, vtype)
    sc, off, qt = oracle.quant_params(vtype, x)
    ones = np.full(n, -1, dtype=np.int64)
    want_ones = expected(oracle, vtype, x, ones, off, sc, qt)
    want = expected(oracle, vtype, x, rowids, off, sc, qt)
    small = np.arange(1, n + 1, dtype=np.int64)
    want_small = expected(oracle, vtype, x, small, off, sc, qt)
    for retain in (n, 0):
        qz = _quantizer(vtype, dim, retain)
        qz.minmax(x)
        src = None if retain else x
        check_bytes(qz.encode(src, ones, off, sc, qt), want_ones, dim, "rowids -1", retain)
        check_bytes(qz.encode(src, small, off, sc, qt), want_small, dim, "rowids 1..n after -1", retain)
        check_bytes(qz.encode(src, rowids, off, sc, qt), want, dim, "extreme rowids", retain)
        qz.close()


# ------------------------------------------------------------------------------------------------ (2) every 16-bit / 8-bit source value
PAIRS = [(0.0, 1.0), (-2.0, 37.5), (0.0, 2.0 ** -8), (0.0, 0.5), (1.5, 0.125), (-3.0, 2.0 ** -12), (0.0, 8.0), (-0.75, 2.0 ** -120)]


def _every_value(vtype):
    if vtype in (po.F16, po.BF16):
        return np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).reshape(2048, 32)
    if vtype == po.U8:
        return np.arange(256, dtype=np.uint8).reshape(16, 16)
    return np.arange(-128, 128, dtype=np.int16).astype(np.int8).reshape(16, 16)


@pytest.mark.parametrize("vtype", [po.F16, po.BF16, po.U8, po.I8])
def test_every_source_value(oracle, vtype):
    """every f16 / bf16 bit pattern (+-0, subnormals, +-Inf, every NaN) and every int8 / uint8 value, both qtypes, with the
    parameters the column itself yields (for f16 / bf16: lo = -Inf, hi = +Inf) and fixed pairs; power-of-two scales put many
    products exactly on a .5 boundary (f16 65408 * 2^-8 = 255.5, 32640 * 2^-8 = 127.5)"""
    x = _every_value(vtype)
    n, dim = x.shape
    rowids = np.arange(n, dtype=np.int64) * 7919 - 5000
    qz = _quantizer(vtype, dim, n)
    qz.minmax(x)
    lo, hi, _ = check_minmax(oracle, qz, vtype, x, "every value")
    for qt in (po.Q_U8, po.Q_S8):
        for off, sc in [params(lo, hi, qt)[::-1]] + PAIRS:
            want = expected(oracle, vtype, x, rowids, off, sc, qt)
            for src in (None, x):
                check_bytes(qz.encode(src, rowids, off, sc, qt), want, dim, vtype, qt, off, sc, src is None)
    qz.close()


# ------------------------------------------------------------------------------------------------ (3) f32 rounding and range edges
F32_PAIRS = [(0.0, 1.0), (0.5, 2.0), (-2.0, 37.5), (0.1, 3.0), (1.0, 0.25), (-7.3, 0.7)]
BIG = [2.0 ** 31 - 256, 2.0 ** 31 - 128, 2.0 ** 31, 2.0 ** 31 + 256, 2.0 ** 32, 1e10, 3e38, FLT_MAX]


def _ulps(x, k):
    with np.errstate(over="ignore"):
        for _ in range(abs(k)):
            x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
    return x


def _fused_disagreements(rng, off, sc, qt, count=4000):
    """f32 inputs near .5 boundaries on which (x - off) * sc rounded twice and fma(x, sc, -off * sc) rounded once give different
    bytes: they tell the two apart"""
    t = rng.integers(-140, 270, count) + 0.5 + rng.uniform(-1e-4, 1e-4, count)
    x = _ulps(np.float32(t / sc + off), 0)
    x = np.concatenate([_ulps(x, k) for k in range(-3, 4)])
    two = q_from_s(po.F32, scaled(po.F32, x, off, sc), qt)
    c = np.float64(np.float32(-np.float32(off) * np.float32(sc)))
    fused = np.float32(x.astype(np.float64) * np.float64(np.float32(sc)) + c)
    return x[two != q_from_s(po.F32, fused, qt)]


@pytest.mark.parametrize("qtype", [po.Q_U8, po.Q_S8])
def test_f32_rounding_and_range_edges(oracle, qtype):
    """f32 sources go through the x86 (int) cast: exact halves k + 0.5 (k = -140..270) and their +-1, +-2 ulp neighbours under
    each (offset, scale) pair, +-0, 254.5 / 255.5 / 126.5 / 127.5 / -127.5 / -128.5, values whose rounded result is just below,
    at and past +-2^31 (INT_MIN: 0 for UINT8 and -128 for INT8, whatever the sign), +-3e38, +-FLT_MAX, +-Inf and NaN"""
    rng = np.random.Generator(np.random.PCG64(77 + qtype))
    targets = np.array([k + 0.5 for k in range(-140, 271)] + [0.0, -0.0, 1e-45, -1e-45, 0.49999997, -0.49999997]
                       + BIG + [-b for b in BIG] + [-(2.0 ** 31)], dtype=np.float64)
    parts = [np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, FLT_MAX, -FLT_MAX, -(2.0 ** 31)], dtype=np.float32)]
    for off, sc in F32_PAIRS:
        with np.errstate(all="ignore"):
            x0 = np.float32(targets / sc + off)
        parts += [_ulps(x0, k) for k in (-2, -1, 0, 1, 2)]
    fused = [_fused_disagreements(rng, off, sc, qtype) for off, sc in F32_PAIRS if (off, sc) != (0.0, 1.0)]
    assert sum(f.size for f in fused) >= 50, "too few inputs tell a fused multiply-add apart"
    x = np.concatenate(parts + fused)
    dim = 13
    x = np.concatenate([x, np.zeros(-x.size % dim, dtype=np.float32)]).reshape(-1, dim)
    n = x.shape[0]
    rowids = np.arange(n, dtype=np.int64) - n // 2
    qz = _quantizer(po.F32, dim, n)
    qz.minmax(x)
    check_minmax(oracle, qz, po.F32, x, "f32 edges")
    for off, sc in F32_PAIRS:
        want = expected(oracle, po.F32, x, rowids, off, sc, qtype)
        for src in (None, x):
            check_bytes(qz.encode(src, rowids, off, sc, qtype), want, dim, off, sc, src is None)
    qz.close()


# ------------------------------------------------------------------------------------------------ (4) the min / max pass
FP_KINDS = ["random", "one_row", "constant", "nonneg", "inf", "pos_inf_only", "neg_inf_only", "nan_only", "nan_mixed", "zeros",
            "empty"]
INT_KINDS = ["random", "one_row", "constant", "nonneg", "empty"]
MINMAX_CASES = [(vt, k) for vt in TYPES for k in (FP_KINDS if vt in (po.F32, po.F16, po.BF16) else INT_KINDS)]


def _minmax_column(vtype, kind, rows, dim, rng):
    """the column in vtype storage; extremes and specials sit in the LAST row, which the block pattern feeds as a one-row tail
    of a staging block"""
    if kind == "one_row":
        rows = 1
    if kind == "empty":
        rows = 0
    if vtype in (po.U8, po.I8):
        lo, hi = (10, 200) if vtype == po.U8 else (-100, 100)
        x = rng.integers(lo, hi, (rows, dim))
        if kind == "random":
            x[-1, dim // 3] = 3 if vtype == po.U8 else -128
            x[-1, dim // 2] = 250 if vtype == po.U8 else 127
        elif kind == "constant":
            x[:] = 7
        elif kind == "nonneg" and vtype == po.I8:
            x = np.abs(x)
        return x.astype(po.NP_STORAGE[vtype])
    x = rng.standard_normal((rows, dim), dtype=np.float32)
    if kind == "empty":
        return po.convert(x, vtype)
    if kind in ("random", "one_row", "nan_mixed", "inf"):
        x[-1, dim // 3], x[-1, dim // 2] = -1000.0, 2000.0
    if kind == "constant":
        x[:] = -2.5
    elif kind == "nonneg":
        x = np.abs(x)
        x[-1, 5] = 0.0
    elif kind == "inf":
        x[-1, 7], x[rows // 2, 9] = np.inf, -np.inf
    elif kind == "pos_inf_only":
        x[:] = np.inf
        x[0, 0] = np.nan
    elif kind == "neg_inf_only":
        x[:] = -np.inf
        x[-1, 1] = np.nan
    elif kind == "nan_only":
        x[:] = np.nan
    elif kind == "nan_mixed":
        x[::3, ::5] = np.nan
        x.view(np.uint32)[1::4, 2::7] = 0xFFC00000          # negative NaN: its order key sits below every number
    elif kind == "zeros":
        x[:] = 0.0
        x[1::2, ::3] = -0.0
    with np.errstate(over="ignore", invalid="ignore"):
        return po.convert(x, vtype)                         # NaN, +-Inf and +-0 keep their class in f16 / bf16


@pytest.mark.parametrize("vtype,kind", MINMAX_CASES)
def test_minmax_pass(oracle, vtype, kind):
    """quant_minmax_kernel and the reduction in minmax_result() against the reference's sequential loop, rows fed in blocks of
    1, S - 1, S and S + 1 rows (S = rows per staging block), retained and streamed.  The loop starts from FLT_MAX / -FLT_MAX
    and updates on `val < lo` / `val > hi`: NaN never enters, an empty or all-NaN column keeps those values, and so does a
    column whose only numbers are +Inf (lo) or -Inf (hi)."""
    rng = np.random.Generator(np.random.PCG64(31 * vtype + len(kind)))
    dim = (1 << 20) // po.ELEM_SIZE[vtype]                  # 1 MiB rows: S = 16
    s = stage_rows(vtype, dim)
    blocks = [1, s - 1, s, s + 1]
    x = _minmax_column(vtype, kind, sum(blocks), dim, rng)
    n = x.shape[0]
    for retain in (n, 0):
        qz = _quantizer(vtype, dim, retain)
        a = 0
        for b in (blocks if n > 1 else [n]):
            qz.minmax(x[a:a + b])
            a += b
        if kind == "empty":
            qz.minmax(x[:0])
        assert a == n
        check_minmax(oracle, qz, vtype, x, kind, retain)
        assert qz.retained_rows == (n if retain else -1)
        qz.close()


# ------------------------------------------------------------------------------------------------ (5) non-finite scales
@pytest.mark.parametrize("vtype", TYPES)
def test_non_finite_scales(oracle, vtype):
    """constant columns (hi - lo = 0: UINT8 scale +Inf), all-zero columns with both signs (scale +Inf for either qtype) and, for
    fp sources, an all-NaN column (UINT8 scale 255 / -Inf = -0.0, offset FLT_MAX): encoded with the derived parameters for
    AUTO and both forced qtypes"""
    rng = np.random.Generator(np.random.PCG64(500 + vtype))
    n, dim = 300, 19
    cols = {"const_pos": np.full((n, dim), 7.0, np.float32), "const_neg": np.full((n, dim), -3.0, np.float32),
            "zeros": np.zeros((n, dim), np.float32)}
    if vtype in (po.F32, po.F16, po.BF16):
        cols["zeros"][::2, 1::2] = -0.0
        cols["nan"] = np.full((n, dim), np.nan, np.float32)
    if vtype == po.U8:
        del cols["const_neg"]
    rowids = rng.integers(INT64_MIN, INT64_MAX, n)
    for name, f in cols.items():
        x = po.convert(f, vtype) if vtype not in (po.U8, po.I8) else f.astype(po.NP_STORAGE[vtype])
        qz = _quantizer(vtype, dim, n)
        qz.minmax(x)
        lo, hi, neg = check_minmax(oracle, qz, vtype, x, name)
        for qt in (po.Q_S8 if neg else po.Q_U8, po.Q_U8, po.Q_S8):
            sc, off = params(lo, hi, qt)
            want = expected(oracle, vtype, x, rowids, off, sc, qt)
            for src in (None, x):
                check_bytes(qz.encode(src, rowids, off, sc, qt), want, dim, name, qt, sc, off, src is None)
        qz.close()


# ------------------------------------------------------------------------------------------------ (6) staging and retention
@pytest.mark.parametrize("vtype", [po.F32, po.BF16])
def test_staging_blocks_and_retention(oracle, vtype):
    """a column of more than three staging blocks (dim 4096: S = 1024 f32 / 2048 bf16 rows per block), fed in blocks of 1,
    S - 1, S, S + 1 and the rest:
      retain_rows = n      retained: whole-column and chunked retained encodes (rows [a, a + m), the last chunk partial, the
                           pattern of rebuild_quantization_gpu), a range past the retained rows or below 0 is VSB_EINVAL;
      retain_rows = 0      streamed;
      retain_rows = n - 1  more rows than announced: nothing retained (-1), encode(None, ...) is VSB_EINVAL;
    and in every case the host rows encode through the two staging buffers with the same bytes."""
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(900 + vtype))
    dim = 4096
    s = stage_rows(vtype, dim)
    n = 3 * s + 77
    xf = rng.standard_normal((n, dim), dtype=np.float32) * 4
    xf[::101, 3] = np.round(xf[::101, 3] * 2) / 2
    xf[-1, 0], xf[s, 1], xf[2 * s + 1, 2] = 90.0, -80.0, np.nan
    x = po.convert(xf, vtype)
    rowids = np.sort(rng.choice(np.arange(-3 * n, 3 * n, dtype=np.int64), n, replace=False)) * 1_000_003
    blocks = [1, s - 1, s, s + 1, n - (3 * s + 1)]
    sc, off, qt = oracle.quant_params(vtype, x)
    want = expected(oracle, vtype, x, rowids, off, sc, qt)
    orow = 8 + dim
    for retain in (n, 0, n - 1):
        qz = _quantizer(vtype, dim, retain)
        a = 0
        for b in blocks:
            qz.minmax(x[a:a + b])
            a += b
        check_minmax(oracle, qz, vtype, x, retain)
        assert qz.retained_rows == (n if retain == n else -1), (retain, qz.retained_rows)
        check_bytes(qz.encode(x, rowids, off, sc, qt), want, dim, "host rows", retain)
        if retain == n:
            check_bytes(qz.encode(None, rowids, off, sc, qt), want, dim, "retained", retain)
            mv = 1000
            for a in range(0, n, mv):
                m = min(mv, n - a)
                got = qz.encode(None, rowids[a:a + m], off, sc, qt, retained_first_row=a)
                check_bytes(got, want[a * orow:(a + m) * orow], dim, "retained chunk", a, m)
            for first, m in ((n - 5, 10), (-1, 4), (n, 1)):
                with pytest.raises(vs.api.VsbError) as e:
                    qz.encode(None, rowids[:m], off, sc, qt, retained_first_row=first)
                assert e.value.rc == vs.api.EINVAL, (first, m, e.value)
        else:
            with pytest.raises(vs.api.VsbError) as e:
                qz.encode(None, rowids[:10], off, sc, qt)
            assert e.value.rc == vs.api.EINVAL, (retain, e.value)
        qz.close()


# ------------------------------------------------------------------------------------------------ (7) vector_quantize through SQL
@needs_ref
@pytest.mark.parametrize("seed", [1, 2, 5, 8, 13, 21])
def test_quantize_fuzz_scripts_on_the_gpu_match_reference(seed):
    """the drawn tables of test_sql_fuzz (5 source types, dims 1..40, NULL rows, NaN / Inf / huge values, constant and
    non-negative columns, negative rowids, both qtypes, several max_memory settings) quantized by the kernels: rows, shadow-table
    bytes, chunk columns and metadata equal the reference statement by statement"""
    script = _quantize_script(seed)
    ours = run_sql(OURS, script, want_launches=True)
    ref = run_sql(REF_CPU, script)
    assert ours[-1]["kernel_launches"] > 0, "vector_quantize did not launch its kernels"
    for s, a, b in zip(script, ours[:-1], ref):
        assert a == b, (seed, s if isinstance(s, str) else s[0], str(a)[:300], str(b)[:300])


def test_small_dim_tables_through_sql(oracle):
    """tables of dims 1..7 with rowids INT64_MIN .. INT64_MAX: vector_quantize on the GPU writes the chunk the oracle builds,
    vector_quantize_scan over it returns the oracle's rowids and distances, and every statement (including the stored scale and
    offset of an all-+Inf and an all--Inf column) equals the host loops' output"""
    rng = np.random.Generator(np.random.PCG64(4242))
    script, checks = [], []
    for d in range(1, 8):
        vt = TYPES[d % 5]
        ids = np.unique(np.concatenate([np.array(ROWIDS + [-(2 ** 40) - 3, 2 ** 62 + 11], dtype=np.int64),
                                        rng.integers(-(2 ** 62), 2 ** 62, 40)]))
        n, k = ids.size, 12
        with np.errstate(over="ignore"):
            x = po.convert(rng.standard_normal((n, d), dtype=np.float32) * 3, vt)
            q = po.convert(rng.standard_normal((1, d), dtype=np.float32) * 3, vt)[0]
        tb = f"t{d}"
        script += [f"CREATE TABLE {tb} (id INTEGER PRIMARY KEY, e BLOB)",
                   f"SELECT vector_init('{tb}', 'e', 'type={TYPE_SQL[vt]},dimension={d},distance=L2')"]
        script += [[f"INSERT INTO {tb}(id, e) VALUES (?, ?)", [int(i), blob(x[r])]] for r, i in enumerate(ids)]
        script += [f"SELECT vector_quantize('{tb}', 'e')", f"SELECT rowid1, rowid2, counter, hex(data) FROM vector0_{tb}_e",
                   f"SELECT key, value FROM _sqliteai_vector WHERE tblname='{tb}' ORDER BY key",
                   [f"SELECT id, distance FROM vector_quantize_scan('{tb}', 'e', ?, {k})", [blob(q)]]]
        checks.append((len(script) - 4, vt, x, ids, q, k))
    for tb, val, opt in (("pinf", np.inf, ""), ("ninf", -np.inf, ", 'qtype=UINT8'")):
        x = np.full((5, 3), val, dtype=np.float32)
        x[2, 1] = np.nan
        script += [f"CREATE TABLE {tb} (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('{tb}', 'e', 'type=FLOAT32,dimension=3')"]
        script += [[f"INSERT INTO {tb}(id, e) VALUES (?, ?)", [int(i) - 2, blob(x[i])]] for i in range(5)]
        script += [f"SELECT vector_quantize('{tb}', 'e'{opt})", f"SELECT hex(data) FROM vector0_{tb}_e",
                   f"SELECT key, value FROM _sqliteai_vector WHERE tblname='{tb}' ORDER BY key"]
    gpu = run_sql(OURS, script, want_launches=True)
    host = run_sql(OURS, script, env={"VSB_QUANTIZE_HOST": "1"}, want_launches=True)
    assert gpu[-1]["kernel_launches"] > host[-1]["kernel_launches"], "vector_quantize did not launch its kernels"
    for s, a, h in zip(script, gpu[:-1], host[:-1]):
        assert a == h, (s if isinstance(s, str) else s[0], a, h)
    for i, vt, x, ids, q, k in checks:
        assert gpu[i] == {"rows": [[ids.size]]}, gpu[i]
        sc, off, qt = oracle.quant_params(vt, x)
        buf = expected(oracle, vt, x, ids, off, sc, qt)
        (row,) = gpu[i + 1]["rows"]
        assert row[:3] == [int(ids[0]), int(ids[-1]), ids.size], row[:3]
        check_bytes(np.frombuffer(bytes.fromhex(row[3]), dtype=np.uint8), buf, x.shape[1], "shadow table", vt)
        qq = oracle.quantize(vt, q, off, sc, qt)
        want_ids, want_d = oracle.scan_quant_buffer(po.L2, qt, qq, buf, ids.size, x.shape[1], k)
        assert gpu[i + 3]["rows"] == [[int(r), float(v)] for r, v in zip(want_ids, want_d)], (vt, x.shape[1])
