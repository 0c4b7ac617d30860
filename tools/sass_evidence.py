"""Which Hopper instructions the built kernels contain: cuobjdump -sass of lib/libvsb200.so, occurrences per kernel.

  python tools/sass_evidence.py > <file>.json
  python tools/sass_evidence.py --compare <parent libvsb200.so> [<libvsb200.so>]

PTX -> SASS names: wgmma.mma_async = HGMMA (f16 / bf16) / IGMMA (s8 / u8), wgmma.fence / commit_group / wait_group = WARPGROUP,
cp.async.bulk.tensor = UTMALDG, cp.async.bulk = UBLKCP, elect.sync = ELECT, dp4a = IDP, redux.sync = REDUX, mbarrier = SYNCS.
HMMA / IMMA (mma.sync) must not appear anywhere.

--compare: every function's whole SASS in two builds, matched by demangled name (addresses and line information stripped), as
JSON: the functions whose code differs, those only in one build, and the count that are identical."""
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WATCH = ("HGMMA", "IGMMA", "WARPGROUP", "UTMALDG", "UBLKCP", "ELECT", "IDP", "REDUX", "HMMA", "IMMA", "SYNCS", "STL", "LDL")
DEFAULT_LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")


def demangle(mangled):
    dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True).stdout.splitlines()
    return {a: b.replace("vsb::", "") for a, b in zip(mangled, dem)}


def sass_by_function(lib):
    """{mangled name: [instruction text, ...]} of every function in lib"""
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    code = collections.defaultdict(list)
    fn = None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(.*?)\s*;", ln)
        if fn is not None and m:
            code[fn].append(m.group(1))
    return code


def compare(old_lib, new_lib):
    old, new = sass_by_function(old_lib), sass_by_function(new_lib)
    on, nn = demangle(sorted(old)), demangle(sorted(new))
    old_d = {on[a]: old[a] for a in old}
    new_d = {nn[a]: new[a] for a in new}
    both = sorted(set(old_d) & set(new_d))
    out = {"how": "whole SASS per function, matched by demangled name (tools/sass_evidence.py --compare)",
           "old": os.path.relpath(old_lib, ROOT), "new": os.path.relpath(new_lib, ROOT),
           "identical": sum(old_d[f] == new_d[f] for f in both),
           "different": [f for f in both if old_d[f] != new_d[f]],
           "only_old": sorted(set(old_d) - set(new_d)),
           "only_new": sorted(set(new_d) - set(old_d))}
    json.dump(out, sys.stdout, indent=1)
    print()


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--compare":
        compare(sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else DEFAULT_LIB)
        return
    lib = sys.argv[1] if len(sys.argv) > 1 else DEFAULT_LIB
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
