"""Recorded answers of the reference's MEX targets -- TEST INFRASTRUCTURE.

The reference MEX targets (oracle/_ref) can only be built where a checkout of the reference is at hand.  So that
the parity tests and smoke() run anywhere, every call they make to the reference is recorded once and stored
under tests/golden/oracle/, one file per caller: the pytest node id of the test, or a name given with
`context(...)` (smoke() uses "smoke").  A call is identified by its position in the caller's sequence; its
inputs are checked against a fingerprint taken when it was recorded (size, sum, sum of squares and a
position-weighted sum, per array), so a recorded answer is never handed to different inputs.

Records are kept small: identical arrays are stored once and float arrays byte-plane shuffled before
compression.  When a record is still larger than RECORD_BUDGET bytes, its large outputs, latest call first, are kept as a
`Sketch` instead -- exact norm, SHA-256 of the bytes and a seeded CountSketch -- one by one until it fits.  A sketched output
can be compared (tests/helpers.py: relerr estimates the relative error from the sketch, exactly 0 when the hashes
agree; same() checks bit equality by hash) and handed back to the reference, but not used in arithmetic.

    SEDUMI_ORACLE=record   call oracle/_ref and (re)write the records of every caller that runs
    SEDUMI_ORACLE=live     call oracle/_ref, ignore the records (timing the reference, new tests)
    (unset)                the record when there is one, else oracle/_ref when it is built
"""
from __future__ import annotations

import atexit
import contextlib
import copy
import hashlib
import json
import os
import re

import numpy as np
import scipy.sparse as sp

from sedumi_b200.mx import MexDir

_HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(_HERE), "tests", "golden", "oracle")
MODE = os.environ.get("SEDUMI_ORACLE", "")

_context = None
_LIVE = object()


@contextlib.contextmanager
def context(name):
    """Key the reference calls made inside the block by `name` instead of the running test."""
    global _context
    old, _context = _context, name
    try:
        yield
    finally:
        _context = old


def _caller():
    if _context is _LIVE:
        return None
    if _context is not None:
        return _context
    t = os.environ.get("PYTEST_CURRENT_TEST")
    return t.rsplit(" (", 1)[0] if t else None


def _path(caller):
    mod, _, name = caller.partition("::")
    mod, name = (os.path.splitext(os.path.basename(mod))[0], name) if name else ("misc", caller)
    name = re.sub(r"[^A-Za-z0-9_.-]+", "_", name)
    return os.path.join(GOLDEN, mod, name + ".npz")


SKETCH_K = 8192                 # CountSketch buckets: relative error of the estimated norm about sqrt(2 / K) = 1.6 %
SKETCH_MIN = 16384              # arrays smaller than this are always stored in full
RECORD_BUDGET = 900_000         # bytes per record file


def _fp(v):
    v = np.asarray(v, dtype=np.float64).ravel(order="F")
    w = ((np.arange(v.size, dtype=np.int64) * 2654435761) % 1000) / 1000.0
    return [float(v.size), float(v.sum()), float((v * v).sum()), float((v * w).sum())]


def _canon(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64).ravel(order="F"))


def _sketch_of(v, k=SKETCH_K):
    rng = np.random.default_rng(v.size)
    idx = rng.integers(0, k, v.size)
    sgn = rng.integers(0, 2, v.size) * 2.0 - 1.0
    return np.bincount(idx, weights=sgn * v, minlength=k)


class Sketch:
    """A large dense output of the reference: shape, exact 2-norm, SHA-256 of its float64 bytes (column-major),
    the fingerprint of its values and a seeded CountSketch of them."""

    def __init__(self, shape, norm, sha, fp, sk):
        self.shape, self.norm, self.sha, self.fp, self.sk = tuple(shape), float(norm), sha, list(fp), sk
        self.size = int(np.prod(self.shape))

    @classmethod
    def of(cls, a):
        v = _canon(a)
        return cls(np.shape(a), np.linalg.norm(v), hashlib.sha256(v.tobytes()).hexdigest(), _fp(v), _sketch_of(v))

    def ravel(self, order="C"):
        return self

    def matches(self, a):
        """True when `a` holds exactly the recorded values."""
        return np.size(a) == self.size and hashlib.sha256(_canon(a).tobytes()).hexdigest() == self.sha

    def error_norm(self, a):
        """||a - recorded||, exact (0) when the bytes agree, else estimated from the sketch."""
        if self.matches(a):
            return 0.0
        return float(np.linalg.norm(_sketch_of(_canon(a)) - self.sk))


class SparseSketch:
    """A large sparse output of the reference: exact pattern, values as a `Sketch`."""

    def __init__(self, indptr, indices, shape, data):
        self.indptr, self.indices, self.shape, self.data = indptr, indices, tuple(shape), data
        self.nnz = int(indptr[-1])


def _arrays(x, out):
    if isinstance(x, dict):
        for k in x:
            _arrays(x[k], out)
    elif isinstance(x, Sketch):
        out.append(x.fp)
    elif isinstance(x, SparseSketch):
        out += [x.data.fp, _fp(x.indices), _fp(x.indptr), _fp(x.shape)]
    elif sp.issparse(x):
        x = sp.csc_matrix(x)
        out += [_fp(x.data), _fp(x.indices), _fp(x.indptr), _fp(np.asarray(x.shape))]
    elif x is not None:
        out.append(_fp(x))
    return out


def fingerprint(args):
    out = []
    for a in args:
        _arrays(a, out)
    return out


def _same_inputs(a, b):
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if x[0] != y[0]:
            return False
        scale = np.sqrt(max(x[2], 0.0) * x[0]) + 1e-300
        if not (abs(x[1] - y[1]) <= 1e-9 * scale and abs(x[2] - y[2]) <= 1e-9 * (x[2] + 1e-300) and abs(x[3] - y[3]) <= 1e-9 * scale):
            return False
    return True


class _Store:
    """Arrays of one record: identical arrays once, float arrays as byte planes (they compress far better)."""

    def __init__(self):
        self.arrays, self.by_hash = {}, {}

    def put(self, a):
        a = np.asarray(a)
        h = hashlib.sha256(a.dtype.str.encode() + str(a.shape).encode() + np.ascontiguousarray(a).tobytes()).hexdigest()
        if h not in self.by_hash:
            key = f"a{len(self.by_hash)}"
            self.by_hash[h] = key
            if a.dtype == np.float64 and a.size:
                self.arrays[key + "@f8"] = np.ascontiguousarray(np.ascontiguousarray(a).reshape(-1).view(np.uint8).reshape(-1, 8).T)
                self.arrays[key + "@shape"] = np.asarray(a.shape, dtype=np.int64)
            else:
                self.arrays[key] = a
        return self.by_hash[h]


def _get(z, key):
    if key + "@f8" in z:
        planes = z[key + "@f8"]
        return np.ascontiguousarray(planes.T).view(np.float64).reshape(tuple(z[key + "@shape"]))
    return z[key].copy()


def _flatten(x, store, sketch):
    """Tree of the output; arrays go to `store`; objects whose id is in `sketch` are kept as sketches."""
    if x is None:
        return {"t": "n"}
    if isinstance(x, dict):
        return {"t": "d", "f": [[k, _flatten(v, store, sketch)] for k, v in x.items()]}
    if sp.issparse(x):
        if not sp.isspmatrix_csc(x):
            x = sp.csc_matrix(x)
        t = {"t": "s", "p": store.put(x.indptr.astype(np.int64)), "i": store.put(x.indices.astype(np.int32)),
             "shape": list(x.shape)}
        if id(x.data) in sketch:
            t["t"], t["k"] = "S", _flatten_sketch(x.data, store)
        else:
            t["v"] = store.put(x.data)
        return t
    if id(x) in sketch:
        return {"t": "k", "k": _flatten_sketch(x, store)}
    return {"t": "a", "v": store.put(x)}


def _flatten_sketch(a, store):
    k = Sketch.of(a)
    return {"shape": list(k.shape), "norm": k.norm, "sha": k.sha, "fp": k.fp, "sk": store.put(k.sk)}


def _sketch_from(t, z):
    return Sketch(t["shape"], t["norm"], t["sha"], t["fp"], _get(z, t["sk"]))


def _unflatten(tree, z):
    t = tree["t"]
    if t == "n":
        return None
    if t == "d":
        return {k: _unflatten(v, z) for k, v in tree["f"]}
    if t == "s":
        return sp.csc_matrix((_get(z, tree["v"]), _get(z, tree["i"]).astype(np.int64), _get(z, tree["p"])),
                             shape=tuple(tree["shape"]))
    if t == "S":
        return SparseSketch(_get(z, tree["p"]), _get(z, tree["i"]).astype(np.int64), tree["shape"], _sketch_from(tree["k"], z))
    if t == "k":
        return _sketch_from(tree["k"], z)
    return _get(z, tree["v"])


def _leaves(x, out):
    """Dense arrays of an output (sparse: the values) -- the candidates for a sketch."""
    if isinstance(x, dict):
        for v in x.values():
            _leaves(v, out)
    elif sp.issparse(x):
        out.append(x.data)
    elif isinstance(x, np.ndarray):
        out.append(x)
    return out


class OracleMissing(ImportError):
    """Neither a record of this call nor the built reference is available."""


class _Recording:
    def __init__(self, caller):
        self.caller = caller
        self.calls = []
        self.replay = None
        if MODE not in ("record", "live") and os.path.exists(_path(caller)):
            with np.load(_path(caller)) as z:
                self.replay = (json.loads(str(z["__calls__"])), {k: z[k] for k in z.files if k != "__calls__"})

    def _write(self, sketch):
        store = _Store()
        calls = [dict(c, out=[_flatten(o, store, sketch) for o in c["out"]]) for c in self.calls]
        np.savez_compressed(_path(self.caller), __calls__=np.array(json.dumps(calls)), **store.arrays)

    def save(self):
        if not self.calls:
            return
        os.makedirs(os.path.dirname(_path(self.caller)), exist_ok=True)
        # latest calls first: what a test hands back to the plugins comes from its earlier reference calls
        cand = [a for c in reversed(self.calls) for o in c["out"] for a in _leaves(o, []) if a.size >= SKETCH_MIN]
        sketch = set()
        self._write(sketch)
        while os.path.getsize(_path(self.caller)) > RECORD_BUDGET and cand:
            sketch.add(id(cand.pop(0)))
            self._write(sketch)


_recordings: dict = {}


@atexit.register
def _save_all():
    if MODE == "record":
        for r in _recordings.values():
            r.save()


def finish(caller):
    """End of a caller: write its record (SEDUMI_ORACLE=record), or check that it used every recorded call -- a
    caller that stops asking the reference part of the way through must not pass against a longer record."""
    rec = _recordings.pop(caller, None)
    if rec is None:
        return
    if MODE == "record":
        rec.save()
    elif rec.replay is not None and len(rec.calls) != len(rec.replay[0]):
        raise AssertionError(f"{caller}: {len(rec.calls)} of {len(rec.replay[0])} recorded reference calls were made")


def has_records(module):
    """True when answers are recorded for tests of `module` (e.g. "test_host")."""
    return os.path.isdir(os.path.join(GOLDEN, module))


def result(inputs, compute):
    """The dict of arrays `compute()` derives from the reference (called live inside it), recorded as one answer of
    the running caller and checked against the fingerprint of `inputs`.  For comparisons whose per-call record would
    be too large: a whole reference iteration at full size."""
    caller = _caller()
    if caller is None or MODE == "live":
        return compute()
    rec = _recordings.get(caller)
    if rec is None:
        rec = _recordings[caller] = _Recording(caller)
    fp = fingerprint(inputs)
    if rec.replay is not None:
        calls, z = rec.replay
        i = len(rec.calls)
        rec.calls.append(None)
        if i >= len(calls) or calls[i]["fn"] != "result":
            raise AssertionError(f"{caller}: reference answer {i} is not a recorded result; re-record with SEDUMI_ORACLE=record")
        if not _same_inputs(calls[i]["fp"], fp):
            raise AssertionError(f"{caller}: inputs of reference answer {i} differ from the recorded ones")
        return _unflatten(calls[i]["out"][0], z)
    with context(_LIVE):
        out = compute()
    if MODE == "record":
        rec.calls.append({"fn": "result", "nlhs": 1, "fp": fp, "out": [copy.deepcopy(out)]})
    return out


class _Target:
    def __init__(self, odir, name):
        self.odir, self.name = odir, name

    def __call__(self, *args, nlhs=1):
        caller = _caller()
        rec = None
        if caller is not None and MODE != "live":
            rec = _recordings.get(caller)
            if rec is None:
                rec = _recordings[caller] = _Recording(caller)
        if rec is not None and rec.replay is not None:
            calls, z = rec.replay
            i = len(rec.calls)
            rec.calls.append(None)
            if i >= len(calls) or calls[i]["fn"] != self.name or calls[i]["nlhs"] != nlhs:
                raise AssertionError(f"{caller}: reference call {i} ({self.name}) is not the recorded one; re-record "
                                     f"with SEDUMI_ORACLE=record")
            if not _same_inputs(calls[i]["fp"], fingerprint(args)):
                raise AssertionError(f"{caller}: inputs of reference call {i} ({self.name}) differ from the recorded ones")
            outs = [_unflatten(t, z) for t in calls[i]["out"]]
            return outs[0] if nlhs <= 1 else tuple(outs)
        if not self.odir.live.has(self.name):
            raise OracleMissing(f"no recorded answer for {self.name} in {caller!r} and oracle/_ref is not built")
        res = getattr(self.odir.live, self.name)(*args, nlhs=nlhs)
        if rec is not None and MODE == "record":
            outs = [res] if nlhs <= 1 else list(res)
            rec.calls.append({"fn": self.name, "nlhs": nlhs, "fp": fingerprint(args), "out": copy.deepcopy(outs)})  # callers may modify res
        return res


class OracleDir:
    """`MexDir` of the reference targets with recorded answers: `OracleDir().blkchol(...)`."""

    def __init__(self, debug=False):
        self.live = MexDir(os.path.join(_HERE, "_ref", "dbg") if debug else os.path.join(_HERE, "_ref"))

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return _Target(self, name)

    def mex_seconds(self):
        """Time spent inside the reference's mexFunctions so far (zero for recorded answers)."""
        return self.live.mex_seconds()

    def has(self, name):
        return self.live.has(name)


def available():
    """True when the reference can be called live (oracle/_ref built)."""
    return MexDir(os.path.join(_HERE, "_ref")).has("blkchol")
