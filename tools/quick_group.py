"""Throughput of the single-query scan on a SMALL shard (default 1.25M x 384 int8 = 1/8 of the bench corpus, what one of 8 GPUs
holds): groups of 8 queries per engine call, one scan launch per query, on one or two scan streams (scan_streams).
Device-timed (CUDA events on the filter stream), filters included, no host copies."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sqlite_vector_b200 as vs  # noqa: E402
from sqlite_vector_b200 import api  # noqa: E402
from tools.quick_bench import make_corpus  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=1_250_000)
ap.add_argument("--dim", type=int, default=384)
ap.add_argument("--queries", type=int, default=1600)
a = ap.parse_args()
eng = vs.load_engine()
ix = vs.Index(api.I8, a.dim, a.n)
make_corpus(ix, api.I8, a.n, a.dim)
pitch = ix.query_pitch
qs = torch.randint(-60, 60, (64, pitch), dtype=torch.int8, device="cuda").view(torch.uint8)
qs[:, a.dim:] = 0
torch.cuda.synchronize()
st = torch.cuda.ExternalStream(ix.stream)
nslots = ix.stat("slots")
G = 8
for streams in (1, 2):
    eng.set_option("scan_streams", streams)

    def run(count):
        grp = 0
        for g0 in range(0, count, G):
            ix.scan_submit_group(api.L2, qs[(g0 % 56)].data_ptr(), pitch, G, 20, True, grp * G, fetch=False)
            grp = (grp + 1) % (nslots // G)
    run(20 * G)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    run(a.queries)
    e1.record(st)
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / a.queries * 1e3
    print(f"scan_streams={streams}: {us:.1f} us/query -> {a.n * a.dim / us / 1e3:.0f} GB/s, {1e6 / us:.0f} q/s per GPU")
eng.set_option("scan_streams", 2)
