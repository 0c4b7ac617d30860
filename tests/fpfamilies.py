"""Adversarial f32 / f16 / bf16 inputs: where an accumulator that truncates, or that aligns its addends to the largest one,
would leave the error model of tc_fp_eps (|s_tc - s| <= dim * 2^-21 * sum |q_i r_i|), and where the FMA chains of the
single-query scan would leave theirs (tests/test_gpu_scan_kernel.py).

make(family, vtype, n, dim, rng) returns the column in storage form (float32, or uint16 bit patterns); decode() widens it to
float64, where every product of two f16 / bf16 values is exact.  Every family has some all-zero rows (row 0 and every 61st),
so the model's demand of an exact 0 is tested everywhere.

"huge" (bf16 and f32 only) puts 0 to 2 elements of magnitude 2^60 .. 2^125 into each row: sums of squares of such rows
overflow fp32 while their root does not.  Exponents 62..64 are left out, so that with a query of ordinary magnitude every
sum of squares, every sum of |d| and every root lies at least a factor 2 away from FLT_MAX: the overflow class of a row does
not depend on rounding."""
import numpy as np

from oracle import pyoracle as po

FAMILIES = ("normal", "wide", "cancel", "dominant", "tiny")   # "huge": see make()


def decode(vtype, a: np.ndarray) -> np.ndarray:
    if vtype == po.F32:
        return np.asarray(a, dtype=np.float32).astype(np.float64)
    a = np.ascontiguousarray(a, dtype=np.uint16)
    if vtype == po.F16:
        return a.view(np.float16).astype(np.float64)
    return (a.astype(np.uint32) << np.uint32(16)).view(np.float32).astype(np.float64)


def _signs(rng, shape):
    return np.where(rng.random(shape) < 0.5, -1.0, 1.0)


def make(family: str, vtype: int, n: int, dim: int, rng: np.random.Generator, queries: bool = False, span: int = 56) -> np.ndarray:
    """queries=True: the query side of the family (for "cancel" both halves equal, so that <row, query> cancels).
    span: bf16 "wide" exponents in [-span, span]"""
    if family == "normal":
        x = rng.standard_normal((n, dim))
    elif family == "wide":
        # +-2^e over as wide a range as keeps every product AND every sum of up to 4096 products finite and normal in
        # fp32: bf16 e in [-56, 56] (products 2^-112 .. 2^112), f16 its whole normal range [-14, 15]
        lo, hi = (-14, 15) if vtype == po.F16 else (-span, span)
        x = _signs(rng, (n, dim)) * np.exp2(rng.integers(lo, hi + 1, (n, dim))).astype(np.float64)
    elif family == "cancel":
        # rows [a, -a'] with a' = a except for a few elements, queries [b, b]: s is a small residue of large terms
        h = dim // 2
        a = rng.standard_normal((n, h)) * np.exp2(rng.integers(-8, 9, (n, 1)))
        b = a.copy()
        nudge = rng.random((n, h)) < 0.125
        b[nudge] *= 1.0 + 2.0 ** -5
        x = np.zeros((n, dim))
        x[:, :h] = a
        x[:, h:2 * h] = -b
        if queries:
            x[:, h:2 * h] = a
    elif family == "dominant":
        # one element per row carries the magnitude, the rest are 2^-10 smaller
        x = rng.standard_normal((n, dim)) * 2.0 ** -10
        j = rng.integers(0, dim, n)
        x[np.arange(n), j] = _signs(rng, n) * (1.0 + rng.random(n))
    elif family == "tiny":
        if vtype == po.F16:                          # f16 subnormals: bit patterns 0x0001 .. 0x03FF, random sign
            bits = rng.integers(1, 0x400, (n, dim)).astype(np.uint16)
            bits |= (rng.random((n, dim)) < 0.5).astype(np.uint16) << np.uint16(15)
            bits[0] = 0
            bits[::61] = 0
            return bits
        # bf16: the smallest magnitudes whose products stay normal in fp32 (2^-63 .. 2^-50 squared >= 2^-126)
        x = _signs(rng, (n, dim)) * np.exp2(rng.integers(-63, -49, (n, dim))).astype(np.float64)
    elif family == "huge":
        if vtype == po.F16:
            raise ValueError("f16 has no huge values")
        x = rng.standard_normal((n, dim))
        exps = np.setdiff1d(np.arange(60, 125), [62, 63, 64])
        for m in (1, 2):
            rows = np.flatnonzero(rng.integers(0, 3, n) >= m)       # 0, 1 or 2 huge elements per row
            cols = rng.integers(0, dim, rows.size)
            mant = 1.0 + rng.integers(0, 128, rows.size) / 128.0      # 8 significant bits: exact in bf16
            x[rows, cols] = _signs(rng, rows.size) * mant * np.exp2(rng.choice(exps, rows.size).astype(np.float64))
    else:
        raise ValueError(family)
    out = po.convert(x.astype(np.float32), vtype)
    out[0] = 0
    out[::61] = 0
    return out
