"""Recorded outputs of the unmodified reference build (oracle/_ref) for exactly the inputs the differential tests draw.

Where oracle/_ref is built the tests call the reference live; everywhere else they compare against what it returned for the
same inputs, stored in tests/golden/ref_<variant>.json.gz (keyed by a digest of the call and its arguments).  Regenerate the
stores where oracle/_ref is built:

    VS_RECORD_REF=1 python -m pytest -m "not gpu" tests/test_oracle_fuzz.py tests/test_oracle_vs_reference.py \
        tests/test_sql_fuzz.py tests/test_sql_surface.py

A call the store does not hold (the test's inputs changed) fails instead of passing silently.
"""
import atexit
import base64
import gzip
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD = os.environ.get("VS_RECORD_REF") == "1"
_stores = {}


def _key(*parts) -> str:
    h = hashlib.blake2b(digest_size=10)
    for p in parts:
        if isinstance(p, np.ndarray):
            a = np.ascontiguousarray(p)
            h.update(f"{a.dtype.str}{a.shape}".encode())
            h.update(a.tobytes())
        elif isinstance(p, np.generic):
            h.update(p.dtype.str.encode())
            h.update(p.tobytes())
        else:
            h.update(repr(p).encode())
        h.update(b"|")
    return h.hexdigest()


def _enc(r):
    if isinstance(r, tuple):
        return ["t", [_enc(x) for x in r]]
    if isinstance(r, np.ndarray):
        return ["a", r.dtype.str, list(r.shape), base64.b64encode(np.ascontiguousarray(r).tobytes()).decode()]
    if isinstance(r, np.generic):
        return ["g", r.dtype.str, base64.b64encode(r.tobytes()).decode()]
    return ["p", r]


def _dec(e):
    if e[0] == "t":
        return tuple(_dec(x) for x in e[1])
    if e[0] == "a":
        return np.frombuffer(base64.b64decode(e[3]), dtype=np.dtype(e[1])).reshape(e[2]).copy()
    if e[0] == "g":
        return np.frombuffer(base64.b64decode(e[2]), dtype=np.dtype(e[1]))[0]
    return e[1]


class _Store:
    def __init__(self, name):
        self.path = os.path.join(GOLDEN, f"ref_{name}.json.gz")
        self.data = {}
        if os.path.exists(self.path):
            with gzip.open(self.path, "rt") as f:
                self.data = json.load(f)
        if RECORD:
            atexit.register(self.save)

    def save(self):
        with gzip.GzipFile(self.path, "wb", mtime=0) as f:
            f.write(json.dumps(self.data, sort_keys=True, separators=(",", ":")).encode())


def store(name) -> _Store:
    if name not in _stores:
        _stores[name] = _Store(name)
    return _stores[name]


def recorded(name, key, live):
    """live(): the reference call, or None where the reference is not built.  Returns its result, live or recorded."""
    st = store(name)
    if live is not None:
        r = live()
        if RECORD:
            st.data[key] = _enc(r)
        return r
    if key not in st.data:
        raise AssertionError(f"no recorded reference output for this input in {os.path.relpath(st.path)}: "
                             "regenerate with VS_RECORD_REF=1 where oracle/_ref is built")
    return _dec(st.data[key])


def available(name) -> bool:
    return bool(store(name).data)


class _Calls:
    def __init__(self, variant, live, prefix):
        self._variant, self._live, self._prefix = variant, live, prefix

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        fn = getattr(self._live, name) if self._live is not None else None

        def call(*args, **kwargs):
            flat = [self._prefix + name, *args]
            for kv in sorted(kwargs.items()):
                flat += list(kv)
            return recorded(self._variant, _key(*flat), None if fn is None else (lambda: fn(*args, **kwargs)))
        return call


class Reference(_Calls):
    """RefHarness(variant) of oracle/pyoracle.py, live when oracle/_ref is built, else replayed from the store."""

    def __init__(self, variant, live):
        super().__init__(variant, live, "")
        self.lib = _Calls(variant, None if live is None else live.lib, "lib.")
        self.backend = recorded(variant, "backend", None if live is None else (lambda: live.backend))


def reference(variant):
    """the reference harness, or None when it is neither built here nor recorded"""
    from oracle import pyoracle
    live = pyoracle.RefHarness(variant) if pyoracle.have_ref() else None
    if live is None and not available(variant):
        return None
    return Reference(variant, live)
