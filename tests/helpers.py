"""Shared test helpers: the two plugin directories and small problem builders.

`ref`  = the UNMODIFIED reference MEX targets compiled into oracle/_ref (the oracle), answered from the
         records under tests/golden/oracle where one exists (oracle/replay.py),
`dbg`  = the same with mxAssert active (validates what our host code marshals when called live),
`gpu`  = the CUDA plugins (sedumi_b200/mex), which fail loudly without a CUDA device.
"""
import os
import sys

import numpy as np
import scipy.sparse as sp

from sedumi_b200.mx import MexDir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import refpath  # noqa: E402
import replay  # noqa: E402

ref = refpath.ref_dir()
dbg = refpath.ref_dir(debug=True)
gpu = MexDir(os.path.join(ROOT, "sedumi_b200", "mex"))

CHOL_PARS = {"canceltol": 1e-12, "maxu": 5e5, "abstol": 1e-20}      # checkpars.m:150-170


def needs_reference(module, target):
    """Skip unless the reference can answer: oracle/_ref built, or answers recorded for the test module."""
    import pytest
    return pytest.mark.skipif(not (ref.has(target) or replay.has_records(module)),
                              reason="oracle/_ref not built and no recorded answers")


def relerr(a, b):
    """||a - b|| / ||b||; b may be a recorded reference output kept as a sketch (oracle/replay.py), then the
    numerator is estimated from the sketch (exactly 0 when a holds the recorded bytes)."""
    if isinstance(b, replay.Sketch):
        a = np.asarray(a.todense() if sp.issparse(a) else a, dtype=float)
        assert a.size == b.size, (a.shape, b.shape)
        return b.error_norm(a if a.shape == b.shape else a.ravel()) / (b.norm if b.norm > 0 else 1.0)
    a = np.asarray(a.todense() if sp.issparse(a) else a, dtype=float)
    b = np.asarray(b.todense() if sp.issparse(b) else b, dtype=float)
    if a.shape != b.shape:                       # (N,1) against (N,): compare element by element, never broadcast
        assert a.size == b.size, (a.shape, b.shape)
        a, b = a.ravel(), b.ravel()
    nb = np.linalg.norm(b)
    return np.linalg.norm(a - b) / (nb if nb > 0 else 1.0)


def same(a, b):
    """Bit equality of two arrays; b may be a recorded reference output kept as a sketch (compared by SHA-256)."""
    if isinstance(b, replay.Sketch):
        return b.matches(a)
    return np.size(a) == np.size(b) and np.array_equal(np.ravel(a, order="F"), np.ravel(b, order="F"))


def dense_L(m):
    """The reference's dense shortcut structure (symbchol.m:75-77)."""
    return {"perm": np.arange(1, m + 1, dtype=float).reshape(-1, 1),
            "L": sp.csc_matrix(np.tril(np.ones((m, m)))),
            "xsuper": np.array([[1.0], [m + 1.0]]), "tmpsiz": 0.0}


def random_spd(m, seed, cond=1e3, rank=None):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((m, m)))
    ev = 10.0 ** rng.uniform(0, np.log10(cond), m)
    if rank is not None:
        ev[rank:] = 0.0
    X = (Q * ev) @ Q.T
    return (X + X.T) / 2


def random_sparse_spd(m, density, seed, shift=None):
    rng = np.random.default_rng(seed)
    A = sp.random(m, m, density=density, random_state=np.random.RandomState(seed), format="csc")
    A = A + A.T
    d = np.asarray(abs(A).sum(axis=1)).ravel() + (1.0 if shift is None else shift)
    X = sp.csc_matrix(A + sp.diags(d * (1 + rng.random(m))))
    X.sort_indices()
    return X


def full_pattern(X):
    """CSC with every entry of a dense matrix stored (what getsymbada gives for dense ADA)."""
    X = np.asarray(X)
    m = X.shape[0]
    return sp.csc_matrix((X.ravel(order="F"), np.tile(np.arange(m), m), np.arange(0, m * m + 1, m)), shape=(m, m))


def check_chol(L, X, pars, absd, tol=1e-10):
    """Run oracle and CUDA blkchol on the same inputs and compare all four outputs."""
    args = (L, X, pars) if absd is None else (L, X, pars, absd)
    LLr, dr, skr, adr = ref.blkchol(*args, nlhs=4)
    LLg, dg, skg, adg = gpu.blkchol(*args, nlhs=4)
    assert np.array_equal(LLr.indptr, LLg.indptr) and np.array_equal(LLr.indices, LLg.indices)
    assert np.array_equal(skr.indices, skg.indices), (skr.indices, skg.indices)
    assert np.array_equal(adr.indices, adg.indices), (adr.indices, adg.indices)
    eL = relerr(LLg.data, LLr.data)
    ed = np.abs(dg - dr).max() / max(np.abs(dr).max(), 1e-300)
    assert eL <= tol, f"L rel err {eL}"
    assert ed <= tol, f"d rel err {ed}"
    if skr.nnz:
        # skipped pivots are cancellation residue: compare on the scale of the matrix
        scale = np.abs(X.diagonal()).max()
        assert np.abs(skg.data - skr.data).max() <= 1e-10 * scale
    if adr.nnz:
        assert relerr(adg.data, adr.data) <= 1e-8
    return (LLr, dr, skr, adr), (LLg, dg, skg, adg)
