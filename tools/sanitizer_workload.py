"""Small invocations of every kernel family for compute-sanitizer (memcheck / racecheck): single-query scans (staged + DIRECT,
k <= 32 and generic filters, all-distances), group launches, the tensor-core batch path (int8 + bf16), sharded merge."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sqlite_vector_b200 as vs  # noqa: E402
from sqlite_vector_b200 import api  # noqa: E402

eng = vs.load_engine()
rng = np.random.Generator(np.random.PCG64(3))


def index(vtype, x):
    ix = vs.Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x)
    ix.finalize()
    return ix


x = rng.integers(-20, 21, (30000, 96)).astype(np.int8)
ix = index(api.I8, x)
q = rng.integers(-20, 21, (40, 96)).astype(np.int8)
for metric in (api.L2, api.COSINE, api.DOT, api.L1):
    for k in (5, 32, 100):
        ix.scan_topk(metric, q[0], k)
ix.scan_all(api.L2, q[0])
ix.scan_submit_group(api.L2, np.ascontiguousarray(q[:8]), q.strides[0], 8, 20, False, 0, fetch=True)
for j in range(8):
    ix.collect(j, 20)
ix.scan_topk(api.L2, q, 20)          # tensor-core batch path (int8)
ix.close()
xb = (rng.standard_normal((20000, 200)).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
ixb = index(api.BF16, xb)
ixb.scan_topk(api.DOT, xb[:32].copy(), 10)
ixb.scan_topk(api.L2, xb[0].copy(), 10)
ixb.close()
# f16 DOT, k = 1: row 5 holds +Inf against all-positive queries, so every query's only slot is -Inf after level 0 and the
# later levels start from max_index 0
xh = rng.standard_normal((20000, 64)).astype(np.float16).view(np.uint16)
xh[5, 0] = 0x7C00
qh = (np.abs(rng.standard_normal((32, 64))) + 0.5).astype(np.float16).view(np.uint16)
ixh = index(api.F16, xh)
ixh.scan_topk(api.DOT, qh, 1)
ixh.close()
xw = rng.standard_normal((600, 20000)).astype(np.float32)     # DIRECT kernel (rows larger than the staging ring)
ixw = index(api.F32, xw)
ixw.scan_topk(api.L2, xw[3].copy(), 7)
ixw.close()
print("workload ok, launches", eng.kernel_launches())
