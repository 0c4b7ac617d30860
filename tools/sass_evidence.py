"""Which Hopper instructions the built kernels contain: cuobjdump -sass of lib/libvsb200.so, occurrences per kernel.

  python tools/sass_evidence.py > <file>.json

PTX -> SASS names: wgmma.mma_async = HGMMA (f16 / bf16) / IGMMA (s8 / u8), wgmma.fence / commit_group / wait_group = WARPGROUP,
cp.async.bulk.tensor = UTMALDG, cp.async.bulk = UBLKCP, elect.sync = ELECT, dp4a = IDP, redux.sync = REDUX, mbarrier = SYNCS.
HMMA / IMMA (mma.sync) must not appear anywhere."""
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WATCH = ("HGMMA", "IGMMA", "WARPGROUP", "UTMALDG", "UBLKCP", "ELECT", "IDP", "REDUX", "HMMA", "IMMA", "SYNCS", "STL", "LDL")


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    names = {}
    counts = collections.defaultdict(collections.Counter)
    fn = None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            fn = m.group(1)
            continue
        if fn is None:
            continue
        m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m:
            op = m.group(1)
            if op in WATCH:
                counts[fn][op] += 1
    mangled = sorted(counts)
    dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True).stdout.splitlines()
    for a, b in zip(mangled, dem):
        names[a] = re.sub(r"\(.*$", "", b).replace("vsb::", "")
    out = {"how": __doc__.split("\n\n")[0] + " (tools/sass_evidence.py)", "library": os.path.relpath(lib, ROOT), "kernels": {}}
    for a in mangled:
        out["kernels"][names[a]] = dict(sorted(counts[a].items()))
    out["kernels_with_wgmma"] = sorted(k for k, v in out["kernels"].items() if "HGMMA" in v or "IGMMA" in v)
    out["kernels_with_tma"] = sorted(k for k, v in out["kernels"].items() if "UTMALDG" in v or "UBLKCP" in v)
    out["mma_sync_anywhere"] = any("HMMA" in v or "IMMA" in v for v in out["kernels"].values())
    out["local_memory_spills"] = sorted(k for k, v in out["kernels"].items() if "STL" in v or "LDL" in v)
    json.dump(out, sys.stdout, indent=1)
    print()


if __name__ == "__main__":
    main()
