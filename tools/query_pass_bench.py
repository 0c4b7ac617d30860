"""Kernel time of one pass of the single-query scan at pass widths nq = 1, 2, 4: scan_kernel alone, one launch at a time on one
stream (scan_streams = 1), CUDA events around each launch (time_kernels), k = 20 L2, device queries through
vsb_scan_submit_group (one pass per nq queries).  A pass reads the column once whatever nq is, so the time per query should
fall close to 1/nq while the pass stays HBM-bound.  Writes one JSON document (card, power limit and max SM clock read in the
same job) to --out."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sqlite_vector_b200 as vs  # noqa: E402
from sqlite_vector_b200 import api  # noqa: E402
from tools.quick_bench import make_corpus  # noqa: E402

SHAPES = [("int8", api.I8, 384, 1), ("f32", api.F32, 384, 4), ("bf16", api.BF16, 768, 2)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def pass_times(eng, ix, dim, k, widths, passes):
    pitch = ix.query_pitch
    qs = torch.zeros((64, pitch), dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(4321)
    q = torch.randn((64, dim), generator=g, device="cuda", dtype=torch.float32)
    if ix.vtype == api.I8:
        qs[:, :dim] = torch.clamp(torch.round(q * 24.0), -128, 127).to(torch.int8).view(torch.uint8)
    elif ix.vtype == api.F32:
        qs[:, :dim * 4] = q.contiguous().view(torch.uint8)
    else:
        qs[:, :dim * 2] = q.to(torch.bfloat16).contiguous().view(torch.uint8)
    torch.cuda.synchronize()
    res = {}
    for nq in widths:
        def run(count):
            for i in range(count):
                ix.scan_submit_group(api.L2, qs[(i * nq) % (64 - nq)].data_ptr(), pitch, nq, k, True, 0, fetch=False)
                torch.cuda.synchronize()
        run(3)
        ix.profile_read()
        eng.set_option("time_kernels", 1)
        p0 = ix.stat("scan_passes")
        run(passes)
        eng.set_option("time_kernels", 0)
        prof = ix.profile_read()
        launched = ix.stat("scan_passes") - p0
        ms = prof["scan_ms"] / max(prof["scan_launches"], 1)
        qpp = nq * passes / max(launched, 1)          # below nq where the shape's widest pass (plan_pass_max) is narrower
        res[str(nq)] = {"pass_ms": ms, "ms_per_query": ms / qpp, "passes": launched, "queries_per_pass": qpp,
                        "filter_ms_per_pass": prof["filter_ms"] / max(prof["filter_launches"], 1)}
    for nq in widths:
        res[str(nq)]["vs_lone_pass"] = res[str(nq)]["pass_ms"] / res[str(widths[0])]["pass_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--passes", type=int, default=20)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    eng = vs.load_engine()
    old = eng.set_option("scan_streams", 1)
    doc = {"card": card(), "k": a.k, "metric": "L2", "rows": a.n, "timing": "CUDA events around each scan launch, scan_streams = 1",
           "shapes": {}}
    for name, vt, dim, esz in SHAPES:
        ix = vs.Index(vt, dim, a.n)
        make_corpus(ix, vt, a.n, dim)
        r = pass_times(eng, ix, dim, a.k, [1, 2, 4], a.passes)
        gb = a.n * dim * esz / 1e9
        for v in r.values():
            v["column_gb_per_s"] = gb / (v["pass_ms"] * 1e-3)
        doc["shapes"][f"{name}_{a.n}x{dim}"] = {"plan_pass_max": ix.stat("plan_pass_max"), "plan_log2p": ix.stat("plan_log2p"),
                                                 "plan_nsw": ix.stat("plan_nsw"), "plan_direct": ix.stat("plan_direct"),
                                                 "column_gb": gb, "widths": r}
        print(name, json.dumps(doc["shapes"][f"{name}_{a.n}x{dim}"]), flush=True)
        ix.close()
        torch.cuda.empty_cache()
    eng.set_option("scan_streams", old)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
