"""TEST INFRASTRUCTURE ONLY.  Stored answers of the compiled reference (oracle/_ref), so that the tests
and smoke() compare with the reference on machines where its sources, and therefore oracle/_ref, do
not exist.

`RecordLib` wraps the real ctypes library: every call is made, and what it wrote (arrays behind
numpy pointers, `byref` scalars, changed ctypes arrays such as the baseline flags) is stored together
with its return value and a fingerprint of its inputs.  `ReplayLib` stands in for the library: the
n-th call of a scope (one test, or smoke()) must name the same function with the same inputs as the
n-th recorded call, and gets the recorded outputs written into its arguments.  Opaque buffers (the
reference's me_data_t, persistent LBFGS state) are neither stored nor checked.

Recordings live in tests/golden/ref/<test module>/<hash of the test id>.npz; `DIRAC_REF_RECORD=<dir>` switches from
replaying to recording into <dir> (needs oracle/_ref, i.e. the reference sources at build time).
"""
from __future__ import annotations

import atexit
import ctypes as C
import json
import os
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")
RECORD_DIR = os.environ.get("DIRAC_REF_RECORD")
SAMPLE_OVER, SAMPLE_N = 1 << 16, 4096   # large dense answers are stored as a sample
MAX_FILE_BYTES = 1000000                 # no stored file above 1 MB

_scope_override = None


def set_scope(name):
    """calls outside pytest (smoke()) are filed under `name`"""
    global _scope_override
    _scope_override = name


def current_scope() -> str:
    if _scope_override:
        return _scope_override
    t = os.environ.get("PYTEST_CURRENT_TEST", "unscoped").rsplit(" (", 1)[0]
    # test ids are relative to pytest's rootdir, which depends on how pytest was started
    path, _, rest = t.partition("::")
    return os.path.basename(path) + "::" + rest


def _group(scope: str) -> str:
    """file a scope is stored in: one per test module"""
    return os.path.splitext(scope.split("::", 1)[0])[0]


def _fingerprint(args):
    fp = []
    for a in args:
        arr = getattr(a, "_arr", None)
        if isinstance(arr, np.ndarray) and arr.dtype.kind in "fc":
            v = arr.view(np.float64) if arr.dtype.kind == "c" else arr
            fp.append([float(v.size), float(np.sum(v)), float(np.sum(np.abs(v)))])
        elif isinstance(arr, np.ndarray):
            fp.append([float(arr.size), float(zlib.crc32(np.ascontiguousarray(arr).tobytes()))])
        elif _blob(a) is not None and not _has_pointers(type(a)):
            fp.append([float(zlib.crc32(bytes(a)))])
        elif isinstance(a, (bool, int, float)) and not _is_address(a):
            fp.append([float(a)])
        elif isinstance(a, C.c_double):
            fp.append([float(a.value)])
    return fp


_CArg = type(C.byref(C.c_int()))


def _is_address(a) -> bool:
    """a raw pointer passed as an integer (`arr.ctypes.data`): what it points to cannot be tracked"""
    return isinstance(a, int) and not isinstance(a, bool) and abs(a) >= 1 << 24


def _has_pointers(t) -> bool:
    """ctypes type whose bytes hold addresses (the sky model): not comparable from run to run"""
    if issubclass(t, C.Array):
        return _has_pointers(t._type_)
    if issubclass(t, C.Structure):
        return any(_has_pointers(ft) for _, ft in t._fields_)
    return issubclass(t, (C._Pointer, C.c_void_p, C.c_char_p))


def _same_fp(got, want):
    """inputs equal to the recorded ones; an input that is itself a sampled replay (NaN) is not checked"""
    if len(got) != len(want):
        return False
    for g, w in zip(got, want):
        if len(g) != len(w):
            return False
        if np.isnan(g).any():
            continue
        if not np.allclose(g, w, rtol=1e-8, atol=1e-300):
            return False
    return True


def _blob(a):
    """ctypes array / structure whose bytes are comparable (not an opaque char buffer)"""
    if isinstance(a, C.Structure) or (isinstance(a, C.Array) and a._type_ is not C.c_char):
        return a
    return None


def _scope_file(scope: str) -> str:
    import hashlib
    return os.path.join(_group(scope), hashlib.sha1(scope.encode()).hexdigest()[:16] + ".npz")


class _Store:
    def __init__(self):
        self.scopes = {}   # scope -> {"calls": [...], "arrays": {key: ndarray}} (None: not stored)
        self.counters = {}
        self.unstorable = set()

    def scope(self, scope, create=False):
        if scope not in self.scopes:
            path = os.path.join(GOLDEN, _scope_file(scope))
            if RECORD_DIR:
                self.scopes[scope] = {"calls": [], "arrays": {}}
            elif os.path.exists(path):
                z = np.load(path, allow_pickle=False)
                self.scopes[scope] = {"calls": json.loads(str(z["index"])),
                                      "arrays": {k: z[k] for k in z.files if k != "index"}}
            else:
                self.scopes[scope] = None
        return self.scopes[scope]

    def next_call(self, scope):
        n = self.counters.get(scope, 0)
        self.counters[scope] = n + 1
        return n

    def save(self, out_dir):
        """one file per scope, tests/golden/ref/<module>/<hash of the test id>.npz; a scope whose file
        would exceed MAX_FILE_BYTES (the dense Jacobians of the larger normal-equation cases) is not
        kept"""
        for scope, d in self.scopes.items():
            if d is None or not d["calls"] or scope in self.unstorable:
                continue
            path = os.path.join(out_dir, _scope_file(scope))
            os.makedirs(os.path.dirname(path), exist_ok=True)
            np.savez_compressed(path, index=np.array(json.dumps(d["calls"])), **d["arrays"])
            if os.path.getsize(path) > MAX_FILE_BYTES:
                os.remove(path)   # runs against the compiled reference where it is built


def _store_array(arrays, a):
    """an output array as stored: whole, or, when it is large and dense (more than SAMPLE_OVER
    elements, less than half of them zero), a fixed seeded sample of SAMPLE_N of its elements; the
    replay leaves the other elements NaN"""
    flat = a.reshape(-1)
    key = "a%d" % len(arrays)
    if a.dtype.kind in "fc" and flat.size > SAMPLE_OVER and np.count_nonzero(flat) > flat.size // 2:
        idx = np.sort(np.random.default_rng(flat.size).choice(flat.size, SAMPLE_N, replace=False))
        arrays[key] = flat[idx].copy()
        arrays[key + "i"] = idx.astype(np.int64)
        return "sample", key
    arrays[key] = a.copy()
    return "arr", key


# element-beam tables filled in by set_elementcoeffs(_wb): scalar fields and the arrays behind the
# pointers are stored, the replay points the structure at copies of them
def _ec_tables(ec, name):
    nf = ec.Nf if name.endswith("_wb") else 1
    dp = C.POINTER(C.c_double)
    return {f: np.ctypeslib.as_array(C.cast(getattr(ec, f), dp), shape=(n,)).copy()
            for f, n in (("pattern_phi", 2 * ec.Nmodes * nf), ("pattern_theta", 2 * ec.Nmodes * nf),
                         ("preamble", ec.Nmodes))}


_store = _Store()
if RECORD_DIR:
    atexit.register(lambda: _store.save(RECORD_DIR))


class _RecordFn:
    def __init__(self, lib_name, fn):
        object.__setattr__(self, "_fn", fn)
        object.__setattr__(self, "_name", lib_name)
        object.__setattr__(self, "real", fn)

    def __setattr__(self, k, v):
        setattr(self._fn, k, v)

    def __getattr__(self, k):
        return getattr(self._fn, k)

    def __call__(self, *args):
        scope = current_scope()
        before = []
        for a in args:
            arr = getattr(a, "_arr", None)
            if isinstance(arr, np.ndarray):
                before.append(arr.copy())
            elif _blob(a) is not None:
                before.append(bytes(a))
            elif isinstance(a, _CArg) and isinstance(a._obj, C.Structure):
                before.append(bytes(a._obj))
            else:
                before.append(None)
        fp = _fingerprint(args)
        if any(_is_address(a) for a in args):
            _store.unstorable.add(scope)
        rv = self._fn(*args)
        d = _store.scope(scope)
        _store.next_call(scope)
        outs = []
        for i, a in enumerate(args):
            arr = getattr(a, "_arr", None)
            if isinstance(arr, np.ndarray):
                if arr.tobytes() != before[i].tobytes():
                    kind, key = _store_array(d["arrays"], arr)
                    outs.append([i, kind, key])
            elif isinstance(a, _CArg):
                obj = a._obj
                if hasattr(obj, "value"):
                    outs.append([i, "byref", float(obj.value)])
                elif self._name.startswith("set_elementcoeffs"):
                    keys = {}
                    for f, t in _ec_tables(obj, self._name).items():
                        keys[f] = "a%d" % len(d["arrays"])
                        d["arrays"][keys[f]] = t
                    keys.update(M=obj.M, Nmodes=obj.Nmodes, Nf=obj.Nf, beta=obj.beta)
                    outs.append([i, "elementcoeff", keys])
                elif bytes(obj) != before[i]:
                    _store.unstorable.add(scope)  # a structure the call filled in
            elif before[i] is not None and bytes(a) != before[i]:
                key = "a%d" % len(d["arrays"])
                d["arrays"][key] = np.frombuffer(bytes(a), dtype=np.uint8).copy()
                outs.append([i, "bytes", key])
        if isinstance(rv, C.Structure):   # returned by value (complex double)
            ret = {"struct": "a%d" % len(d["arrays"])}
            d["arrays"][ret["struct"]] = np.frombuffer(bytes(rv), dtype=np.uint8).copy()
        else:
            ret = rv if isinstance(rv, (int, float)) or rv is None else None
        d["calls"].append({"fn": self._name, "fp": fp, "ret": ret, "outs": outs})
        return rv


class RecordLib:
    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = _RecordFn(name, getattr(self._lib, name))
        self.__dict__[name] = fn
        return fn


def _recorded(scope) -> bool:
    return _store.scope(scope) is not None


class _ReplayFn:
    def __init__(self, owner, name):
        object.__setattr__(self, "_owner", owner)
        object.__setattr__(self, "_name", name)
        object.__setattr__(self, "_types", {})

    def __setattr__(self, k, v):
        self._types[k] = v  # argtypes / restype, for the live library

    @property
    def real(self):
        return self._live_fn() if not _recorded(current_scope()) else C.c_void_p(0)

    def _live_fn(self):
        fn = getattr(self._owner.live(), self._name)
        for k, v in self._types.items():
            setattr(fn, k, v)
        return fn

    def __call__(self, *args):
        scope = current_scope()
        if not _recorded(scope) or any(_is_address(a) for a in args):
            return self._live_fn()(*args)
        d = _store.scope(scope)
        n = _store.next_call(scope)
        calls = d["calls"]
        if n >= len(calls):
            raise AssertionError("no recorded reference answer for call %d (%s) of %s; record it with "
                                 "DIRAC_REF_RECORD (tests/golden/ref)" % (n, self._name, scope))
        c = calls[n]
        if c["fn"] != self._name or not _same_fp(_fingerprint(args), c["fp"]):
            raise AssertionError("call %d of %s: %s with these inputs was not recorded (recorded: %s)"
                                 % (n, scope, self._name, c["fn"]))
        for i, kind, val in c["outs"]:
            a = args[i]
            if kind == "arr":
                a._arr[...] = d["arrays"][val].reshape(a._arr.shape)
            elif kind == "sample":
                flat = a._arr.reshape(-1)
                flat[...] = np.nan
                flat[d["arrays"][val + "i"]] = d["arrays"][val]
            elif kind == "byref":
                a._obj.value = val
            elif kind == "elementcoeff":
                ec = a._obj
                ec._tables = {f: d["arrays"][val[f]].copy() for f in ("pattern_phi", "pattern_theta",
                                                                       "preamble")}
                for f, t in ec._tables.items():
                    setattr(ec, f, t.ctypes.data)
                ec.M, ec.Nmodes, ec.Nf, ec.beta = val["M"], val["Nmodes"], val["Nf"], val["beta"]
            else:
                src = d["arrays"][val].tobytes()
                C.memmove(C.addressof(a), src, len(src))
        if isinstance(c["ret"], dict):
            return self._types["restype"].from_buffer_copy(d["arrays"][c["ret"]["struct"]].tobytes())
        return c["ret"]


class ReplayLib:
    """recorded answers where the scope was stored; otherwise the compiled library at `live_path`
    when it exists (a test that has not been recorded), else the test is skipped"""

    def __init__(self, live_path):
        self._live_path = live_path
        self._live = None

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        fn = _ReplayFn(self, name)
        self.__dict__[name] = fn
        return fn

    def live(self):
        if self._live is None:
            if not os.path.exists(self._live_path):
                import pytest
                pytest.skip("the reference's answers for %s are not stored and %s is not built "
                            "(make -C oracle with the reference sources)"
                            % (current_scope(), os.path.relpath(self._live_path, ROOT)))
            self._live = C.CDLL(self._live_path, mode=C.RTLD_GLOBAL)
        return self._live
