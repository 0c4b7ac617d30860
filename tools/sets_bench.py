"""Per-query eligible sets (vsb_scan_topk_sets, DESIGN §3.14) on one H100.

Workload: int8 --n x 384 (seeded), L2, k = 20, a batch of 1024 queries, and these set families:
  - random10: 1024 distinct random 10 % sets (each a random word rotation of one of 16 random bitmaps);
  - random1: the same at 1 %;
  - tenant_blocks: 16 tenants owning contiguous blocks of rows, 64 queries each;
  - tenant_random: 16 tenants owning a random partition of the rows, 64 queries each;
  - bf16_dot768_random10: a bf16 dim-768 column of --bf16-n rows, DOT, with 1024 random 10 % sets.
Per family: the median time of the sets call, the upload of its bitmaps alone (pageable host -> device, as the call does),
sets_plan_us / sets_levels / fallbacks of the call, the same queries set by set through vsb_scan_topk_filtered, the unfiltered
batch, whether every answer equals the set-by-set answer bit for bit (expected for int8; fp single calls round differently
from the batch refine), and whether 16 sampled answers equal the filtered batch over the same queries under their set.  Reads the card's name, power limit and clocks in the
same run.  Writes profiles/h100_sets.json (or --out).

    python tools/sets_bench.py [--n 10000000] [--bf16-n 4000000] [--reps 3] [--out profiles/h100_sets.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sqlite_vector_b200 as vs  # noqa: E402
from sqlite_vector_b200 import api  # noqa: E402

K, B, T = 20, 1024, 16


def _smi():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def _ms(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def _column(vtype, n, dim, seed, chunk=1 << 20):
    ix = vs.Index(vtype, dim, n)
    rng = np.random.Generator(np.random.PCG64(seed))
    for a in range(0, n, chunk):
        m = min(chunk, n - a)
        if vtype == api.I8:
            ix.append_dense(rng.integers(-64, 64, (m, dim), dtype=np.int8))
        else:
            ix.append_dense((rng.standard_normal((m, dim), dtype=np.float32).view(np.uint32) >> 16).astype(np.uint16))
    ix.finalize()
    return ix


def _queries(vtype, nq, dim, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    if vtype == api.I8:
        return rng.integers(-64, 64, (nq, dim), dtype=np.int8)
    return (rng.standard_normal((nq, dim), dtype=np.float32).view(np.uint32) >> 16).astype(np.uint16)


def _random_sets(n, frac, count, rng):
    words = (n + 31) // 32
    base = [api.row_bitmap(rng.random(n) < frac) for _ in range(16)]
    out = np.zeros((count, words), np.uint32)
    for i in range(count):
        out[i] = np.roll(base[i % 16], int(rng.integers(0, words)))
    if n % 32:
        out[:, -1] &= np.uint32((1 << (n % 32)) - 1)
    return out


def _tenant_sets(n, blocks, rng):
    owner = (np.arange(n) * T // n) if blocks else rng.integers(0, T, n)
    return np.stack([api.row_bitmap(owner == t) for t in range(T)])


def _family(ix, metric, q, sets, soq, reps):
    """one family: timings, counters and the set-by-set comparison"""
    import torch
    out = {}
    flat = np.ascontiguousarray(sets)
    torch.cuda.synchronize()
    ups = []
    for _ in range(reps):
        t0 = time.perf_counter()
        d = torch.from_numpy(flat.view(np.int32)).to("cuda")
        torch.cuda.synchronize()
        ups.append((time.perf_counter() - t0) * 1e3)
        del d
    out["upload_ms"] = sorted(ups)[len(ups) // 2]
    out["bitmap_bytes"] = int(flat.nbytes)
    ix.scan_topk_sets(metric, q, K, flat, soq, as_arrays=True)        # warm-up
    times, got = [], None
    for _ in range(reps):
        b0, f0, p0 = ix.stat("sets_batches"), ix.stat("sets_fallbacks"), ix.stat("sets_plan_us")
        ms, got = _ms(lambda: ix.scan_topk_sets(metric, q, K, flat, soq, as_arrays=True))
        times.append(ms)
        out["one_pass"] = ix.stat("sets_batches") - b0 == 1
        out["fallbacks"] = ix.stat("sets_fallbacks") - f0
        out["sets_plan_us"] = ix.stat("sets_plan_us") - p0
        out["sets_levels"] = ix.stat("sets_levels")
    out["sets_call_ms"] = sorted(times)[len(times) // 2]
    out["sets_call_ms_all"] = times
    # set by set: one filtered call per distinct set over its queries
    t0 = time.perf_counter()
    same = True
    for s in sorted(set(soq.tolist())):
        idx = np.flatnonzero(soq == s)
        want = ix.scan_topk_filtered(metric, q[idx], K, flat[s], as_arrays=True)
        for j, b in enumerate(idx):
            c = int(want[2][j])
            same &= int(got[2][b]) == c and np.array_equal(got[0][b, :c], want[0][j, :c]) and \
                np.array_equal(got[1][b, :c].view(np.uint64), want[1][j, :c].view(np.uint64))
    out["set_by_set_ms"] = (time.perf_counter() - t0) * 1e3
    out["equal_to_set_by_set"] = bool(same)
    # the one-pass answer of query b equals the filtered batch over the SAME queries under b's set (fp batches round like the
    # refine, not like single calls); checked on 16 sampled queries
    same = True
    for b in range(0, q.shape[0], max(1, q.shape[0] // 16)):
        want = ix.scan_topk_filtered(metric, q, K, flat[soq[b]], as_arrays=True)
        c = int(want[2][b])
        same &= int(got[2][b]) == c and np.array_equal(got[0][b, :c], want[0][b, :c]) and \
            np.array_equal(got[1][b, :c].view(np.uint64), want[1][b, :c].view(np.uint64))
    out["equal_to_filtered_batch_sampled"] = bool(same)
    ix.scan_topk(metric, q, K, as_arrays=True)
    un = [_ms(lambda: ix.scan_topk(metric, q, K, as_arrays=True))[0] for _ in range(reps)]
    out["unfiltered_batch_ms"] = sorted(un)[len(un) // 2]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--bf16-n", type=int, default=4_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sets.json"))
    a = ap.parse_args()
    res = {"gpu": _smi(), "n": a.n, "dim": 384, "k": K, "batch": B}
    rng = np.random.Generator(np.random.PCG64(77))
    ix = _column(api.I8, a.n, 384, 1)
    q = _queries(api.I8, B, 384, 2)
    fams = {}
    every = np.arange(B, dtype=np.int32)
    tenants = (np.arange(B) // (B // T)).astype(np.int32)
    fams["random10"] = _family(ix, api.L2, q, _random_sets(a.n, 0.10, B, rng), every, a.reps)
    print("random10", fams["random10"], flush=True)
    fams["random1"] = _family(ix, api.L2, q, _random_sets(a.n, 0.01, B, rng), every, a.reps)
    print("random1", fams["random1"], flush=True)
    fams["tenant_blocks"] = _family(ix, api.L2, q, _tenant_sets(a.n, True, rng), tenants, a.reps)
    print("tenant_blocks", fams["tenant_blocks"], flush=True)
    fams["tenant_random"] = _family(ix, api.L2, q, _tenant_sets(a.n, False, rng), tenants, a.reps)
    print("tenant_random", fams["tenant_random"], flush=True)
    ix.close()
    if a.bf16_n > 0:
        bx = _column(api.BF16, a.bf16_n, 768, 3)
        bq = _queries(api.BF16, B, 768, 4)
        fams["bf16_dot768_random10"] = _family(bx, api.DOT, bq, _random_sets(a.bf16_n, 0.10, B, rng), every, a.reps)
        fams["bf16_dot768_random10"]["n"] = a.bf16_n
        print("bf16", fams["bf16_dot768_random10"], flush=True)
        bx.close()
    res["families"] = fams
    res["gpu_after"] = _smi()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
