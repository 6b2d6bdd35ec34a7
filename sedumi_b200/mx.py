"""ctypes marshalling between numpy/scipy objects and mxshim ``mxArray``s.

This is the host side of the MEX boundary when no MATLAB/Octave interpreter is
present: Python plays the interpreter's role and calls ``mexFunction`` in a plugin
``.so`` exactly as MATLAB would (SURVEY.md section 8b; reference plugins e.g.
blkchol.c:239, getada3.c:370).  The same marshalling drives both the CUDA plugins in
``sedumi_b200/mex/`` and (in tests / the CPU baseline only) the reference plugins in
``oracle/_ref/``.

Conventions (mirror MATLAB):
  * numpy float arrays  -> full double matrices, column-major; 1-D arrays become
    column vectors (m x 1) unless ``row=True``.
  * scipy.sparse        -> CSC sparse double; explicit zeros are PRESERVED (the ADA
    chain relies on stored zeros, getada1.c:222-225).
  * dict                -> 1x1 struct.
  * python scalars      -> 1x1 double.
"""
from __future__ import annotations

import ctypes as C
import os
import time
from typing import Any, Sequence

import numpy as np
import scipy.sparse as sp

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SHIM_PATH = os.path.join(_ROOT, "mxshim", "libmxshim.so")

_shim = None


class MexError(RuntimeError):
    """Raised when a plugin calls mexErrMsgTxt (or a debug mxAssert fails)."""


def shim() -> C.CDLL:
    global _shim
    if _shim is None:
        if not os.path.exists(_SHIM_PATH):
            raise ImportError(
                f"{_SHIM_PATH} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
        lib = C.CDLL(_SHIM_PATH, mode=C.RTLD_GLOBAL)
        vp, sz, dbl = C.c_void_p, C.c_size_t, C.c_double
        lib.mxCreateDoubleMatrix.restype = vp
        lib.mxCreateDoubleMatrix.argtypes = [sz, sz, C.c_int]
        lib.mxCreateSparse.restype = vp
        lib.mxCreateSparse.argtypes = [sz, sz, sz, C.c_int]
        lib.mxCreateStructMatrix.restype = vp
        lib.mxCreateStructMatrix.argtypes = [sz, sz, C.c_int, C.POINTER(C.c_char_p)]
        lib.mxDestroyArray.argtypes = [vp]
        lib.mxDestroyArray.restype = None
        for f in ("mxGetPr", "mxGetJc", "mxGetIr"):
            getattr(lib, f).restype = vp
            getattr(lib, f).argtypes = [vp]
        for f in ("mxGetM", "mxGetN", "mxGetNzmax"):
            getattr(lib, f).restype = sz
            getattr(lib, f).argtypes = [vp]
        lib.mxshim_class.restype = C.c_int
        lib.mxshim_class.argtypes = [vp]
        lib.mxSetField.argtypes = [vp, sz, C.c_char_p, vp]
        lib.mxSetField.restype = None
        lib.mxGetField.restype = vp
        lib.mxGetField.argtypes = [vp, sz, C.c_char_p]
        lib.mxGetNumberOfFields.restype = C.c_int
        lib.mxGetNumberOfFields.argtypes = [vp]
        lib.mxGetFieldNameByNumber.restype = C.c_char_p
        lib.mxGetFieldNameByNumber.argtypes = [vp, C.c_int]
        lib.mxshim_call.restype = C.c_int
        lib.mxshim_call.argtypes = [vp, C.c_int, C.POINTER(vp), C.c_int, C.POINTER(vp)]
        lib.mxshim_last_error.restype = C.c_char_p
        _shim = lib
    return _shim


def _copy_in(ptr: int, arr: np.ndarray) -> None:
    if arr.size:
        C.memmove(ptr, arr.ctypes.data, arr.nbytes)


def to_mx(obj: Any) -> int:
    """Build an mxArray (returned as an integer address) from a Python object."""
    lib = shim()
    if isinstance(obj, dict):
        names = list(obj.keys())
        arr_t = C.c_char_p * max(len(names), 1)
        cn = arr_t(*[n.encode() for n in names])
        s = lib.mxCreateStructMatrix(1, 1, len(names), cn)
        for n in names:
            lib.mxSetField(s, 0, n.encode(), to_mx(obj[n]))
        return s
    if sp.issparse(obj):
        a = obj if sp.isspmatrix_csc(obj) else sp.csc_matrix(obj)
        if not a.has_sorted_indices:
            a = a.copy()
            a.sort_indices()
        m, n = a.shape
        nnz = int(a.indptr[-1])
        x = lib.mxCreateSparse(m, n, max(nnz, 1), 0)
        _copy_in(lib.mxGetJc(x), np.ascontiguousarray(a.indptr, dtype=np.uint64))
        _copy_in(lib.mxGetIr(x), np.ascontiguousarray(a.indices[:nnz], dtype=np.uint64))
        _copy_in(lib.mxGetPr(x), np.ascontiguousarray(a.data[:nnz], dtype=np.float64))
        return x
    a = np.asarray(obj, dtype=np.float64)
    if a.ndim == 0:
        a = a.reshape(1, 1)
    elif a.ndim == 1:
        a = a.reshape(-1, 1)
    elif a.ndim != 2:
        raise ValueError("only <=2-D arrays cross the MEX boundary")
    m, n = a.shape
    x = lib.mxCreateDoubleMatrix(m, n, 0)
    _copy_in(lib.mxGetPr(x), np.asfortranarray(a))
    return x


def _as_np(ptr: int, count: int, dtype) -> np.ndarray:
    if count == 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    ct = C.c_double if dtype == np.float64 else C.c_uint64
    buf = (ct * count).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=count).copy()


def from_mx(x: int) -> Any:
    """Convert an mxArray back to numpy / scipy.sparse / dict (copies the data)."""
    lib = shim()
    if not x:
        return None
    cls = lib.mxshim_class(x)
    m, n = lib.mxGetM(x), lib.mxGetN(x)
    if cls == 2:
        out = {}
        for i in range(lib.mxGetNumberOfFields(x)):
            name = lib.mxGetFieldNameByNumber(x, i)
            out[name.decode()] = from_mx(lib.mxGetField(x, 0, name))
        return out
    if cls == 1:
        jc = _as_np(lib.mxGetJc(x), n + 1, np.uint64).astype(np.int64)
        nnz = int(jc[-1]) if n > 0 else 0
        ir = _as_np(lib.mxGetIr(x), nnz, np.uint64).astype(np.int64)
        pr = _as_np(lib.mxGetPr(x), nnz, np.float64)
        a = sp.csc_matrix((pr, ir, jc), shape=(m, n))
        return a
    return _as_np(lib.mxGetPr(x), m * n, np.float64).reshape((m, n), order="F")


def free_mx(x: int) -> None:
    if x:
        shim().mxDestroyArray(x)


class MexPlugin:
    """One ``<target>.so`` exporting ``mexFunction`` (install_sedumi.m:70-110)."""

    def __init__(self, path: str):
        shim()
        if not os.path.exists(path):
            raise ImportError(f"MEX plugin not built: {path}")
        self.path = path
        self.lib = C.CDLL(path)
        self.fn = C.cast(self.lib.mexFunction, C.c_void_p)
        self.seconds = 0.0          # time spent inside mexFunction (marshalling excluded)
        self.calls = 0

    def call_raw(self, nlhs: int, prhs: Sequence[int]) -> list[int]:
        """Call with pre-built mxArray inputs; returns raw output handles (caller frees)."""
        lib = shim()
        nout = max(nlhs, 1)
        plhs = (C.c_void_p * nout)()
        rhs = (C.c_void_p * max(len(prhs), 1))(*prhs)
        t0 = time.perf_counter()
        rc = lib.mxshim_call(self.fn, nlhs, plhs, len(prhs), rhs)
        self.seconds += time.perf_counter() - t0
        self.calls += 1
        if rc != 0:
            raise MexError(lib.mxshim_last_error().decode(errors="replace"))
        return [plhs[i] for i in range(nout)]

    def __call__(self, *args: Any, nlhs: int = 1):
        prhs = [to_mx(a) for a in args]
        try:
            outs = self.call_raw(nlhs, prhs)
            res = [from_mx(o) for o in outs]
            for o in outs:
                free_mx(o)
        finally:
            for p in prhs:
                free_mx(p)
        return res[0] if nlhs <= 1 else tuple(res[:nlhs])


class MexDir:
    """Attribute access to the plugins in one directory: ``MexDir(path).blkchol(...)``."""

    def __init__(self, path: str):
        self.path = path
        self._cache: dict[str, MexPlugin] = {}

    def __getattr__(self, name: str) -> MexPlugin:
        if name.startswith("_"):
            raise AttributeError(name)
        if name not in self._cache:
            self._cache[name] = MexPlugin(os.path.join(self.path, name + ".so"))
        return self._cache[name]

    def mex_seconds(self) -> float:
        """Total time spent inside the plugins' mexFunction so far."""
        return sum(p.seconds for p in self._cache.values())

    def has(self, name: str) -> bool:
        return os.path.exists(os.path.join(self.path, name + ".so"))
